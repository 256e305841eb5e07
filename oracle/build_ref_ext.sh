#!/bin/bash
# oracle/build_ref_ext.sh — TEST INFRASTRUCTURE.  Installs the reference's OWN PyTorch extensions, unmodified and
# through their own setup.py (torch.utils.cpp_extension, i.e. the stock build path: rasterize_points.cu + ext.cpp,
# torch caching allocator, current-stream semantics as upstream), for sm_90a into oracle/_ref/site/:
#     diff_gaussian_rasterization (+ _C)   from $REF/submodules/diff-gaussian-rasterization
#     simple_knn (+ _C)                    from $REF/submodules/simple-knn   (needs <cfloat>: NVCC_APPEND_FLAGS)
# The source trees are read-only, so pip builds from a scratch copy under /tmp.  Nothing is copied into the repo:
# oracle/_ref/ is git-ignored (it travels to the GPU box with the gpurun snapshot like our own built .so files).
# bench.py --impl reference and the rasterizer parity tests import the result via oracle/ref_ext.py.
set -euo pipefail
REF=${REF:-/root/reference}
HERE=$(cd "$(dirname "$0")" && pwd)
OUT=$HERE/_ref/site
if [ ! -d "$REF/submodules/diff-gaussian-rasterization" ]; then
  echo "build_ref_ext: $REF not present, keeping prebuilt $OUT (if any)"; exit 0
fi
if [ -f "$OUT/diff_gaussian_rasterization/__init__.py" ] && ls "$OUT"/diff_gaussian_rasterization/_C*.so >/dev/null 2>&1 \
   && ls "$OUT"/simple_knn/_C*.so >/dev/null 2>&1 && [ -z "${FORCE:-}" ]; then
  echo "build_ref_ext: $OUT is up to date"; exit 0
fi
TMP=$(mktemp -d /tmp/ref_ext.XXXXXX)
trap 'rm -rf "$TMP"' EXIT
cp -r "$REF/submodules/diff-gaussian-rasterization" "$TMP/dgr"
cp -r "$REF/submodules/simple-knn" "$TMP/sk"
mkdir -p "$OUT"
export TORCH_CUDA_ARCH_LIST="9.0a" MAX_JOBS=${MAX_JOBS:-8} FORCE_CUDA=1
python -m pip install --no-index --no-build-isolation --no-deps --upgrade --target "$OUT" "$TMP/dgr"
NVCC_APPEND_FLAGS="-include cfloat" python -m pip install --no-index --no-build-isolation --no-deps --upgrade --target "$OUT" "$TMP/sk"
ls -la "$OUT" "$OUT/diff_gaussian_rasterization" "$OUT/simple_knn"
