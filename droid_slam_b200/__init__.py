"""H100-native (sm_90a) dense-BA update hot path of DROID-SLAM behind the reference's `droid_backends` API.

    import droid_slam_b200
    droid_slam_b200.install()        # makes `import droid_backends` resolve to the native extension
    import droid_backends            # same nine callables as princeton-vl/DROID-SLAM src/droid.cpp:246-259

    droid_slam_b200.install_dependencies()   # also `import lietorch` / `import torch_scatter` -> droid_slam_b200.lietorch / .torch_scatter

There is no CPU or PyTorch fallback: if the native extension has not been built (`python -m droid_slam_b200.build`)
`install()` / `backends()` raise ImportError.
"""
import importlib
import os
import sys

__all__ = ["install", "install_dependencies", "backends", "capi", "EXT_DIR", "LIB_PATH"]

_PKG = os.path.dirname(os.path.abspath(__file__))
EXT_DIR = os.path.join(_PKG, "_ext")
LIB_PATH = os.path.join(_PKG, "lib", "libdroid_b200.so")


def install():
    """Put the native `droid_backends` extension first on sys.path and import it (after torch)."""
    import torch  # noqa: F401  (libtorch must be loaded before the extension)
    if EXT_DIR not in sys.path:
        sys.path.insert(0, EXT_DIR)
    mod = importlib.import_module("droid_backends")
    if not getattr(mod, "_b200_native", lambda: False)():
        raise ImportError("a different `droid_backends` module shadows the native one: %r" % (mod,))
    return mod


def install_dependencies():
    """install(), then register this package's `lietorch` (SO3 / SE3 on the native kernels) and `torch_scatter` (scatter_sum /
    scatter_mean) as the top-level modules `lietorch` and `torch_scatter`, so the reference's Python imports without any third-party CUDA
    build.  Raises ImportError when a different `lietorch` or `torch_scatter` is already imported.  Recorded in the hook registry: a
    DroidAsync backend started with `spawn` registers both before its arguments are unpickled (modules.BackendProcess)."""
    mod = install()
    from . import lietorch, modules, torch_scatter
    ours = {"lietorch": lietorch, "torch_scatter": torch_scatter}
    for name, pkg in ours.items():
        have = sys.modules.get(name)
        if have is not None and have is not pkg:
            raise ImportError("a different `%s` module is already imported (%r); install_dependencies would shadow it" % (name, have))
    sys.modules.update(ours)
    modules._record("install_dependencies", sys.modules[__name__])
    return mod


def backends():
    return install()


def capi():
    """ctypes handle on the C ABI (include/droid_b200.h)."""
    from . import c_api
    return c_api.load()
