#!/bin/bash
# TEST/BENCH INFRASTRUCTURE -- compiles the REFERENCE's own CUDA extensions (vendored mamba_ssm
# selective_scan + causal_conv1d, unmodified sources where they lie in the reference checkout, $ZIGMA_REFERENCE_ROOT) for sm_90a
# into oracle/_ref/{selective_scan_cuda,causal_conv1d_cuda}.so, with the reference's own nvcc flags
# (dis_mamba/setup.py:137-156, dis_causal_conv1d/setup.py) and only the -gencode swapped: the shipped
# setup.py files target sm_70/80/90 only (dis_mamba/setup.py:108-114) and carry no sm_90a target.
# Nothing is copied into the repo; the outputs are git-ignored.
# They are the "reference vendored CUDA path" baseline that bench.py times next to our kernels.
set -e
REF=${ZIGMA_REFERENCE_ROOT:-/root/reference}
HERE="$(cd "$(dirname "$0")" && pwd)"
OUT="$HERE/_ref"
OBJ="$OUT/obj"
mkdir -p "$OBJ"
[ -d "$REF/dis_mamba/csrc" ] || { echo "reference not found at $REF"; exit 0; }
if [ -f "$OUT/selective_scan_cuda.so" ] && [ -f "$OUT/causal_conv1d_cuda.so" ] && [ -z "$FORCE" ]; then echo "oracle/_ref up to date"; exit 0; fi
PY=${PYTHON:-python}
INC=$($PY - <<'PYEOF'
import sysconfig, torch.utils.cpp_extension as c
print(" ".join("-I" + p for p in c.include_paths() + [sysconfig.get_paths()["include"]]))
PYEOF
)
TLIB=$($PY -c "import torch, os; print(os.path.join(os.path.dirname(torch.__file__), 'lib'))")
NVCC=${NVCC:-/usr/local/cuda/bin/nvcc}
COMMON="-O3 -std=c++17 -Xcompiler -fPIC -DTORCH_API_INCLUDE_EXTENSION_H -D_GLIBCXX_USE_CXX11_ABI=1 $INC"
NVF="$COMMON -U__CUDA_NO_HALF_OPERATORS__ -U__CUDA_NO_HALF_CONVERSIONS__ -U__CUDA_NO_BFLOAT16_OPERATORS__ -U__CUDA_NO_BFLOAT16_CONVERSIONS__ -U__CUDA_NO_BFLOAT162_OPERATORS__ -U__CUDA_NO_BFLOAT162_CONVERSIONS__ --expt-relaxed-constexpr --expt-extended-lambda --use_fast_math -lineinfo -gencode arch=compute_90a,code=sm_90a -w"
build_ext () {   # name srcdir
    local name=$1 dir=$2; shift 2
    local objs=() pids=()
    for f in "$dir"/*.cu "$dir"/*.cpp; do
        [ -e "$f" ] || continue
        local o="$OBJ/${name}_$(basename "$f").o"
        objs+=("$o")
        [ -f "$o" ] && continue
        ( $NVCC $NVF -DTORCH_EXTENSION_NAME=$name -c "$f" -o "$o" > "$o.log" 2>&1 || { cat "$o.log"; exit 1; } ) &
        pids+=($!)
        while [ $(jobs -r | wc -l) -ge ${JOBS:-6} ]; do sleep 1; done
    done
    for p in "${pids[@]}"; do wait $p; done
    $NVCC -shared -o "$OUT/$name.so" "${objs[@]}" -L"$TLIB" -ltorch -ltorch_cpu -ltorch_cuda -ltorch_python -lc10 -lc10_cuda -lcudart
    echo "built $OUT/$name.so"
}
build_ext causal_conv1d_cuda "$REF/dis_causal_conv1d/csrc"
build_ext selective_scan_cuda "$REF/dis_mamba/csrc/selective_scan"
