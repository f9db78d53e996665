#!/bin/bash
# Build liblvsr_b200.so (sm_90a only) in-tree.  Usage: build.sh [extra nvcc flags]
set -euo pipefail
cd "$(dirname "$0")"
NVCC=${NVCC:-/usr/local/cuda/bin/nvcc}
ARCH="-gencode arch=compute_90a,code=sm_90a"
FLAGS="$ARCH -O3 -lineinfo -std=c++17 -Xcompiler -fPIC -I../../include -I."
# objects built with other flags (another architecture, say) are stale too
STAMP=build.flags
if [ ! -f $STAMP ] || [ "$(cat $STAMP)" != "$FLAGS $*" ]; then
  rm -f ./*.o
  echo "$FLAGS $*" > $STAMP
fi
OBJS=()
for f in gemm gemm_tc bigru bigru_bwd attention decoder dec_scan bottom train noise stats search lm fbank tle api; do
  stale=0
  for h in kernels.h common.cuh attention_row.cuh model.h train_kernels.cuh ../../include/lvsr_b200.h; do
    if [ "$h" -nt "$f.o" ]; then stale=1; fi
  done
  if [ ! -f "$f.o" ] || [ "$f.cu" -nt "$f.o" ] || [ $stale = 1 ]; then
    echo "nvcc $f.cu"
    $NVCC $FLAGS "$@" -c "$f.cu" -o "$f.o"
  fi
  OBJS+=("$f.o")
done
$NVCC $ARCH -shared -o liblvsr_b200.so "${OBJS[@]}" -lcudart
echo "built $(pwd)/liblvsr_b200.so"
