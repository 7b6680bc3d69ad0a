#!/usr/bin/env bash
# Builds the UNMODIFIED reference CUDA rasterizer/voxelizer (6 .cu files, compiled from where they
# lie in the reference checkout, R2_REFERENCE_ROOT or /root/reference) + oracle/ref_shim.cu into oracle/_ref/libr2ref.so
# for sm_90a.  Baseline infrastructure only (golden-vector generation, the bench's reference arm);
# oracle/_ref/ is git-ignored.
# Needs: oracle/glm_standin (the reference's GLM submodule is un-vendored) and -include cstdint
# (RAS/rasterizer_impl.h:24 uses std::uintptr_t without the header).
set -euo pipefail
HERE="$(cd "$(dirname "$0")" && pwd)"
REF="${R2_REFERENCE_ROOT:-/root/reference}"
SUB="$REF/r2_gaussian/submodules/xray-gaussian-rasterization-voxelization"
OUT="$HERE/_ref"
if [ ! -d "$SUB/cuda_rasterizer" ]; then
  echo "build_ref: $SUB not present - keeping prebuilt $OUT" >&2
  exit 0
fi
mkdir -p "$OUT/obj"
NVCC="${NVCC:-/usr/local/cuda/bin/nvcc}"
FLAGS=(-std=c++17 -O3 -gencode arch=compute_90a,code=sm_90a -lineinfo -Xcompiler -fPIC
       -I"$HERE/glm_standin" -I"$SUB" -include cstdint -w)
srcs=(cuda_rasterizer/forward.cu cuda_rasterizer/backward.cu cuda_rasterizer/rasterizer_impl.cu
      cuda_voxelizer/forward.cu cuda_voxelizer/backward.cu cuda_voxelizer/voxelizer_impl.cu)
pids=()
for s in "${srcs[@]}"; do
  o="$OUT/obj/$(echo "$s" | tr '/' '_' | sed 's/\.cu$/.o/')"
  if [ ! -f "$o" ] || [ "$SUB/$s" -nt "$o" ] || [ "$HERE/glm_standin/glm/glm.hpp" -nt "$o" ]; then
    "$NVCC" "${FLAGS[@]}" -c "$SUB/$s" -o "$o" &
    pids+=($!)
  fi
done
o="$OUT/obj/ref_shim.o"
if [ ! -f "$o" ] || [ "$HERE/ref_shim.cu" -nt "$o" ]; then
  "$NVCC" "${FLAGS[@]}" -c "$HERE/ref_shim.cu" -o "$o" &
  pids+=($!)
fi
for p in "${pids[@]:-}"; do [ -n "$p" ] && wait "$p"; done
"$NVCC" -shared -o "$OUT/libr2ref.so" "$OUT"/obj/*.o -lcudart
echo "build_ref: built $OUT/libr2ref.so"
