#!/bin/bash
# Build libnrw.so (sm_90a only) in-tree: neuralrecon-w_b200/nrw/libnrw.so
set -e
HERE="$(cd "$(dirname "$0")" && pwd)"
SRC="$HERE/csrc"
OUT="$HERE/nrw/libnrw.so"
OBJ="$HERE/build"
mkdir -p "$OBJ"
NVCC=${NVCC:-/usr/local/cuda/bin/nvcc}
FLAGS="-gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -std=c++17 -Xcompiler -fPIC,-fvisibility=hidden --expt-relaxed-constexpr"
pids=()
for f in gemm_tc gemm_simt pack pointwise embed sampler composite octree octree_build optim dataio mcubes nnsearch raster raygen voxelvis viewsel engine c_api; do
  if [ ! -f "$OBJ/$f.o" ] || [ "$SRC/$f.cu" -nt "$OBJ/$f.o" ] || [ -n "$(find "$SRC" "$HERE/../include" -name '*.h' -newer "$OBJ/$f.o" -o -name '*.cuh' -newer "$OBJ/$f.o" 2>/dev/null | head -1)" ]; then
    ( $NVCC $FLAGS ${NRW_PTXAS_V:+-Xptxas -v} -c "$SRC/$f.cu" -o "$OBJ/$f.o" 2>&1 | sed "s/^/[$f] /" ; exit ${PIPESTATUS[0]} ) &
    pids+=($!)
  fi
done
rc=0
for p in "${pids[@]}"; do wait $p || rc=1; done
[ $rc -eq 0 ] || { echo "build failed"; exit 1; }
$NVCC -shared -o "$OUT" "$OBJ"/*.o -lcudart_static -lrt -lpthread -ldl
echo "built $OUT"
