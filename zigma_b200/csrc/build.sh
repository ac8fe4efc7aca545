#!/bin/bash
# Builds libzigma_b200.so (sm_90a) in-tree: zigma_b200/lib/libzigma_b200.so
# A translation unit is recompiled when it, one of the headers it includes (nvcc -MMD dependency file) or the C-ABI header changed.
set -e
HERE="$(cd "$(dirname "$0")" && pwd)"
OUT="$HERE/../lib"
OBJ="$HERE/../../build/obj"
mkdir -p "$OUT" "$OBJ"
NVCC=${NVCC:-/usr/local/cuda/bin/nvcc}
FLAGS="-gencode arch=compute_90a,code=sm_90a -lineinfo -O3 -std=c++17 -Xcompiler -fPIC -Xptxas -v"
stale() {   # $1 = object, $2 = source
    [ -f "$1" ] && [ -f "$1.d" ] || return 0
    [ "$2" -nt "$1" ] && return 0
    for dep in $(sed -e 's/^[^:]*://' -e 's/\\$//' "$1.d"); do
        case "$dep" in /usr/*|/opt/*) continue ;; esac
        [ -e "$dep" ] && [ "$dep" -nt "$1" ] && return 0
    done
    return 1
}
pids=()
objs=()     # only the objects of the sources that exist now are linked (build/obj may hold objects of sources since removed)
for f in "$HERE"/*.cu; do
    o="$OBJ/$(basename "${f%.cu}").o"
    objs+=("$o")
    if stale "$o" "$f"; then
        ( $NVCC $FLAGS -MMD -MF "$o.d" -c "$f" -o "$o" > "$o.log" 2>&1 || { cat "$o.log"; rm -f "$o"; exit 1; } ) &
        pids+=($!)
    fi
done
rc=0
for p in "${pids[@]}"; do wait $p || rc=1; done
[ $rc -eq 0 ] || { echo "build failed"; exit 1; }
$NVCC -gencode arch=compute_90a,code=sm_90a -shared -o "$OUT/libzigma_b200.so" "${objs[@]}" -lcudart -lcuda
echo "built $OUT/libzigma_b200.so"
