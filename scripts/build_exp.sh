#!/bin/bash
# builds zigma_b200/lib/libzigma_exp<name>.so with extra nvcc flags for one TU (default scan_fwd_bf16.cu; timing experiments)
#   scripts/build_exp.sh t1 "-DZG_TAIL_PREFETCH_MOD=1" norm.cu
set -e
cd "$(dirname "$0")/.."
name=$1; extra=${2:?usage: build_exp.sh <name> "<nvcc flags>" [<tu.cu>]}; tu=${3:-scan_fwd_bf16.cu}
mkdir -p build/exp/obj$name
FLAGS="-gencode arch=compute_90a,code=sm_90a -lineinfo -O3 -std=c++17 -Xcompiler -fPIC $extra"
for f in zigma_b200/csrc/*.cu; do
  o=build/exp/obj$name/$(basename ${f%.cu}).o
  case $(basename $f) in $tu) nvcc $FLAGS -c $f -o $o & ;; *) cp build/obj/$(basename ${f%.cu}).o $o ;; esac
done
wait
nvcc -gencode arch=compute_90a,code=sm_90a -shared -o zigma_b200/lib/libzigma_exp$name.so build/exp/obj$name/*.o -lcudart -lcuda
echo built zigma_b200/lib/libzigma_exp$name.so
