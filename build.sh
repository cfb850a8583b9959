#!/bin/bash
# Build libyolob200.so (sm_90a) in-tree.  Usage: ./build.sh [extra nvcc flags]
set -e
cd "$(dirname "$0")"
SRC=yolov3_tensorflow_b200/csrc
OUT=yolov3_tensorflow_b200/libyolob200.so
mkdir -p build
NVCC=${NVCC:-/usr/local/cuda/bin/nvcc}
FLAGS="-gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -lineinfo -Xcompiler -fPIC --expt-relaxed-constexpr $*"
# objects compiled with other flags (another architecture, say) are rebuilt
if [ "$(cat build/flags 2>/dev/null)" != "$FLAGS" ]; then rm -f build/*.o; echo "$FLAGS" > build/flags; fi
pids=()
for f in $SRC/*.cu; do
  o=build/$(basename ${f%.cu}).o
  if [ ! -f "$o" ] || [ "$f" -nt "$o" ] || [ -n "$(find $SRC include -newer "$o" \( -name '*.cuh' -o -name '*.h' \) | head -1)" ]; then
    $NVCC $FLAGS -c "$f" -o "$o" &
    pids+=($!)
  fi
done
for p in "${pids[@]}"; do wait $p; done
$NVCC -gencode arch=compute_90a,code=sm_90a -shared -o $OUT build/*.o -cudart static
echo "built $OUT"
