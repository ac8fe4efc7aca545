"""CPU: SASS audit of the wgmma GEMM (zg::gemm_bf16_tn_kernel).  Every instantiation exists, spills nothing to local memory, and
has no GPU-scope memory barrier (MEMBAR.*.GPU) between its first and its last HGMMA: handing a ring stage back to the producers
of the cluster is an mbarrier arrive without a fence, so the main loop never waits for the memory system of the whole GPU."""
import re
import subprocess

import pytest

from test_deterministic_abi import _tool

GPU_MEMBAR = re.compile(r"\bMEMBAR(?:\.[A-Z0-9_]+)*\.GPU\b")
LOCAL_MEM = re.compile(r"\b(?:LDL|STL)(?:\.[A-Z0-9_]+)*\b")


def _gemm_functions():
    cuobjdump, filt = _tool("cuobjdump"), _tool("cu++filt")
    if cuobjdump is None or filt is None:
        pytest.skip("cuobjdump / cu++filt not available")
    import __graft_entry__
    __graft_entry__.build()
    from zigma_b200 import _lib
    sass = subprocess.run([cuobjdump, "-sass", _lib.LIB_PATH], check=True, capture_output=True, text=True).stdout
    funcs, cur = {}, None
    for line in sass.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            cur = m.group(1)
            funcs[cur] = []
        elif cur is not None:
            funcs[cur].append(line)
    names = list(funcs)
    demangled = subprocess.run([filt], input="\n".join(names), check=True, capture_output=True, text=True).stdout.splitlines()
    out = {}
    for mangled, dem in zip(names, demangled):
        m = re.search(r"zg::gemm_bf16_tn_kernel<(.*)>\(", dem)
        if m:
            out[tuple(re.sub(r"^\((?:int|bool)\)", "", a.strip()) for a in m.group(1).split(","))] = funcs[mangled]
    return out


def test_sass_gemm_main_loop_has_no_gpu_scope_fence():
    funcs = _gemm_functions()
    # every tile width the dispatcher picks, each with clusters of 1, 2 and 4 CTAs, except 80-wide tiles in clusters of 4 (a CTA's
    # 20-row multicast slice of the weight tile would not be whole 8-row swizzle groups)
    want = {(bn, cl) for bn in ("64", "80", "128", "160", "256") for cl in ("1", "2", "4")} - {("80", "4")}
    assert want == {k[:2] for k in funcs}, sorted(funcs)
    clustered_fences = 0
    for args, lines in funcs.items():
        mma = [i for i, l in enumerate(lines) if "HGMMA" in l]
        assert mma, f"gemm_bf16_tn_kernel<{', '.join(args)}> has no HGMMA"
        fences = [i for i, l in enumerate(lines) if GPU_MEMBAR.search(l)]
        inside = [lines[i].strip() for i in fences if mma[0] < i < mma[-1]]
        assert not inside, f"gemm_bf16_tn_kernel<{', '.join(args)}>: GPU-scope fence between HGMMAs: {inside[:3]}"
        spills = [l.strip() for l in lines if LOCAL_MEM.search(l)]
        assert not spills, f"gemm_bf16_tn_kernel<{', '.join(args)}> uses local memory: {spills[:3]}"
        if args[1] != "1":
            clustered_fences += len(fences)
    # the pattern does match: the cluster-wide barriers at kernel entry and exit of the clustered instantiations compile to one
    assert clustered_fences > 0
