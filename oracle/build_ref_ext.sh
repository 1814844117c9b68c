#!/usr/bin/env bash
# TEST INFRASTRUCTURE ONLY -- builds the *unmodified* reference PointNet++ op
# library (pvn3d/_ext-src) for sm_90a, straight from the sources where they
# lie under /root/reference, into oracle/_ref/_ext.so.
#
# It is the live GPU oracle for the bit-exactness tests (tests/ -m gpu) and the
# "stock PointNet++ kernels" timing baseline printed by bench.py.  Nothing in
# the product path (pvn3d_b200/) imports it.  oracle/_ref/ is git-ignored.
#
# Recipe = reference setup.py:16-34 (CUDAExtension, "-O2", include dir) done by
# hand, plus ONE define (-DAT_CHECK=TORCH_CHECK) because torch>=1.5 renamed the
# macro used at _ext-src/include/utils.h:5-25.  No source edits.
set -euo pipefail
REF=${REF:-/root/reference/pvn3d/_ext-src}
HERE="$(cd "$(dirname "$0")" && pwd)"
OUT="$HERE/_ref"
if [ ! -d "$REF" ]; then
  echo "[oracle] $REF absent -- keeping prebuilt oracle/_ref" >&2
  exit 0
fi
mkdir -p "$OUT/obj"
# Stage the reference PYTHON the GPU-side tests and bench.py's stock-GPU baseline import (a GPU machine
# may have no reference checkout): lib/ (without the 84 MB ResNet checkpoint), common.py and the keypoint /
# radius text fixtures under datasets/.  Verbatim copies into the git-ignored oracle/_ref/py -- test
# infrastructure, never part of the repository history.
PYREF="$(dirname "$REF")"
if [ -d "$PYREF/lib" ]; then
  rm -rf "$OUT/py"; mkdir -p "$OUT/py"
  tar -C "$PYREF" --exclude='ResNet_pretrained_mdl' --exclude='__pycache__' --exclude='*.pyc' -cf - \
      lib common.py datasets | tar -C "$OUT/py" -xf -
  echo "[oracle] staged reference python under oracle/_ref/py ($(du -sh "$OUT/py" | cut -f1))"
fi
if [ -f "$OUT/_ext.so" ] && [ "$OUT/_ext.so" -nt "$REF/src/sampling_gpu.cu" ] && [ "${FORCE:-0}" != 1 ]; then
  echo "[oracle] oracle/_ref/_ext.so up to date"; exit 0
fi
PY=${PYTHON:-python}
TORCH=$($PY -c 'import torch,os;print(os.path.dirname(torch.__file__))')
PYINC=$($PY -c 'import sysconfig;print(sysconfig.get_paths()["include"])')
TI="-I$REF/include -I$TORCH/include -I$TORCH/include/torch/csrc/api/include -I$PYINC -I/usr/local/cuda/include"
DEFS="-DTORCH_EXTENSION_NAME=_ext -DAT_CHECK=TORCH_CHECK -DTORCH_API_INCLUDE_EXTENSION_H"
pids=()
for f in ball_query group_points interpolate sampling; do
  g++ -std=c++17 -O2 -fPIC $TI $DEFS -c "$REF/src/$f.cpp" -o "$OUT/obj/$f.o" &
  pids+=($!)
  nvcc -std=c++17 -O2 -Xcompiler -fPIC -gencode arch=compute_90a,code=sm_90a \
       $TI $DEFS -c "$REF/src/${f}_gpu.cu" -o "$OUT/obj/${f}_gpu.o" &
  pids+=($!)
done
g++ -std=c++17 -O2 -fPIC $TI $DEFS -c "$REF/src/bindings.cpp" -o "$OUT/obj/bindings.o" &
pids+=($!)
for p in "${pids[@]}"; do wait "$p"; done
g++ -shared -o "$OUT/_ext.so" "$OUT"/obj/*.o \
    -L"$TORCH/lib" -L/usr/local/cuda/lib64 \
    -lc10 -ltorch -ltorch_cpu -ltorch_python -lc10_cuda -ltorch_cuda -lcudart \
    -Wl,-rpath,"$TORCH/lib"
echo "[oracle] built $OUT/_ext.so"
