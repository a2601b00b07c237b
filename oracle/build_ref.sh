#!/usr/bin/env bash
# Build the UNMODIFIED reference droid_backends (src/*.cu, src/droid.cpp read in place from
# /root/reference) for sm_90a as `droid_backends_ref`, against the Eigen stand-in in
# oracle/eigen_standin (Eigen itself is an absent submodule).  Output only into oracle/_ref/.
# This is measurement/test infrastructure: the product never links or imports it.
set -euo pipefail
HERE="$(cd "$(dirname "${BASH_SOURCE[0]}")" && pwd)"
REF="${DROID_REFERENCE_ROOT:-/root/reference}"
OUT="$HERE/_ref"
mkdir -p "$OUT"
if [ ! -d "$REF/src" ]; then echo "reference sources not present at $REF; keeping prebuilt $OUT" >&2; exit 0; fi
PY="${PYTHON:-python}"
read -r TORCH_INC PY_INC TORCH_LIB EXT <<<"$($PY - <<'PYEOF'
import torch, sysconfig, os
ti = os.path.join(os.path.dirname(torch.__file__), "include")
print(ti, sysconfig.get_paths()["include"], os.path.join(os.path.dirname(torch.__file__), "lib"), sysconfig.get_config_var("EXT_SUFFIX"))
PYEOF
)"
NAME=droid_backends_ref
TARGET="$OUT/$NAME$EXT"
COMMON=(-O3 -std=c++17 -DTORCH_EXTENSION_NAME=$NAME -DTORCH_API_INCLUDE_EXTENSION_H -D_GLIBCXX_USE_CXX11_ABI=1
        -I"$HERE/eigen_standin" -I"$TORCH_INC" -I"$TORCH_INC/torch/csrc/api/include" -I"$PY_INC" -I/usr/local/cuda/include)
NVCC=(/usr/local/cuda/bin/nvcc -gencode arch=compute_90a,code=sm_90a -Xcompiler -fPIC --expt-relaxed-constexpr
      -D__CUDA_NO_HALF_OPERATORS__ -D__CUDA_NO_HALF_CONVERSIONS__ -D__CUDA_NO_BFLOAT16_CONVERSIONS__ -D__CUDA_NO_HALF2_OPERATORS__)
stale() { [ ! -f "$1" ] || [ "$2" -nt "$1" ]; }
pids=()
for f in droid_kernels correlation_kernels altcorr_kernel; do
  if stale "$OUT/$f.o" "$REF/src/$f.cu" || stale "$OUT/$f.o" "$HERE/eigen_standin/Eigen/SparseCore" || stale "$OUT/$f.o" "$HERE/eigen_standin/Eigen/SparseCholesky"; then
    "${NVCC[@]}" "${COMMON[@]}" -c "$REF/src/$f.cu" -o "$OUT/$f.o" & pids+=($!)
  fi
done
if stale "$OUT/droid.o" "$REF/src/droid.cpp"; then
  g++ -fPIC "${COMMON[@]}" -c "$REF/src/droid.cpp" -o "$OUT/droid.o" & pids+=($!)
fi
g++ -fPIC "${COMMON[@]}" -c "$HERE/ref_timer.cpp" -o "$OUT/ref_timer.o" & pids+=($!)
for p in "${pids[@]}"; do wait "$p"; done
g++ -shared -o "$TARGET" "$OUT"/droid_kernels.o "$OUT"/correlation_kernels.o "$OUT"/altcorr_kernel.o "$OUT"/droid.o "$OUT"/ref_timer.o \
    -L"$TORCH_LIB" -lc10 -lc10_cuda -ltorch_cpu -ltorch_cuda -ltorch -ltorch_python -L/usr/local/cuda/lib64 -lcudart \
    -Wl,-rpath,"$TORCH_LIB"
echo "built $TARGET"
