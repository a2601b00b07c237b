"""In-tree build of the native code (no JIT cache: the built .so files travel with the repo snapshot).

  lib/libdroid_b200.so                          C-ABI library, hand-written CUDA for sm_90a (nvcc, no torch headers)
  _ext/droid_backends.cpython-*.so              pybind11/torch binding exporting the reference's `droid_backends` API

`python -m droid_slam_b200.build` (or `__graft_entry__.build()`) rebuilds what is stale.
"""
import os
import subprocess
import sys
import sysconfig
from concurrent.futures import ThreadPoolExecutor

PKG = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(PKG, "csrc")
LIBDIR = os.path.join(PKG, "lib")
EXTDIR = os.path.join(PKG, "_ext")
OBJDIR = os.path.join(PKG, "build")
INCLUDE = os.path.join(os.path.dirname(PKG), "include")

CUDA_HOME = os.environ.get("CUDA_HOME", "/usr/local/cuda")
NVCC = os.environ.get("NVCC", os.path.join(CUDA_HOME, "bin", "nvcc"))
CUDA_SOURCES = ["common.cu", "corr_index.cu", "corr_lookup_rows.cu", "altcorr.cu", "geom.cu", "ba.cu", "chol.cu", "corr_volume.cu", "update_op.cu", "encoder.cu", "proximity.cu", "filler.cu", "handover.cu", "lie.cu", "ba_layer.cu", "corr_train.cu"]
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
              "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr", "-diag-suppress", "177"]

LIB_PATH = os.path.join(LIBDIR, "libdroid_b200.so")
EXT_PATH = os.path.join(EXTDIR, "droid_backends" + sysconfig.get_config_var("EXT_SUFFIX"))


def _newer(target, deps):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps)


def _run(cmd):
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("build command failed:\n  %s\n%s\n%s" % (" ".join(cmd), r.stdout, r.stderr))
    return r.stdout + r.stderr


def build_library(verbose=False):
    os.makedirs(LIBDIR, exist_ok=True)
    os.makedirs(OBJDIR, exist_ok=True)
    headers = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))]
    headers += [os.path.join(INCLUDE, "droid_b200.h"), os.path.join(INCLUDE, "droid_b200_training.h")]
    jobs = []
    objs = []
    for src in CUDA_SOURCES:
        s = os.path.join(CSRC, src)
        o = os.path.join(OBJDIR, src.replace(".cu", ".o"))
        objs.append(o)
        if _newer(o, [s] + headers):
            jobs.append([NVCC] + NVCC_FLAGS + ["-c", s, "-o", o])
    if jobs:
        with ThreadPoolExecutor(max_workers=min(8, len(jobs))) as ex:
            for out in ex.map(_run, jobs):
                if verbose and out.strip():
                    print(out)
    if jobs or _newer(LIB_PATH, objs):
        _run([NVCC, "-shared", "-o", LIB_PATH] + objs + ["-gencode", "arch=compute_90a,code=sm_90a", "-lcudart"])
    return LIB_PATH


def build_binding(verbose=False):
    import torch
    os.makedirs(EXTDIR, exist_ok=True)
    src = os.path.join(CSRC, "binding", "droid_backends.cpp")
    if not _newer(EXT_PATH, [src, os.path.join(INCLUDE, "droid_b200.h"), os.path.join(INCLUDE, "droid_b200_training.h"), LIB_PATH]):
        return EXT_PATH
    tdir = os.path.dirname(torch.__file__)
    tinc = os.path.join(tdir, "include")
    tlib = os.path.join(tdir, "lib")
    cmd = ["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-DTORCH_EXTENSION_NAME=droid_backends",
           "-DTORCH_API_INCLUDE_EXTENSION_H", "-D_GLIBCXX_USE_CXX11_ABI=%d" % int(torch._C._GLIBCXX_USE_CXX11_ABI),
           "-I" + tinc, "-I" + os.path.join(tinc, "torch", "csrc", "api", "include"),
           "-I" + sysconfig.get_paths()["include"], "-I" + os.path.join(CUDA_HOME, "include"),
           src, "-o", EXT_PATH,
           "-L" + LIBDIR, "-ldroid_b200", "-L" + tlib, "-lc10", "-lc10_cuda", "-ltorch_cpu", "-ltorch_cuda", "-ltorch",
           "-ltorch_python", "-L" + os.path.join(CUDA_HOME, "lib64"), "-lcudart",
           "-Wl,-rpath,$ORIGIN/../lib", "-Wl,-rpath," + tlib]
    out = _run(cmd)
    if verbose and out.strip():
        print(out)
    return EXT_PATH


def build_all(verbose=False):
    build_library(verbose)
    build_binding(verbose)
    return LIB_PATH, EXT_PATH


if __name__ == "__main__":
    print(build_all(verbose=True))
