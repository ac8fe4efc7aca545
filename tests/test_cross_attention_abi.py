"""CPU: the cross-attention entry points (zg_cross_attn_fwd / _bwd, include/zigma_b200.h) -- ctypes layout of the new
structs, the backward workspace size against the documented segment rule, the argument checks on empty batches (which pass
validation and launch nothing, so no GPU is needed), and a SASS audit: every xattn kernel instantiation exists and none
contains a floating-point atomic or reduction."""
import ctypes
import os
import re
import subprocess
import tempfile

import pytest

from test_deterministic_abi import FLOAT_ATOMIC, _tool

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "zigma_b200.h")
FAKE = 1 << 20            # stands in for device pointers: the checks read addresses, never memory


def _built():
    import __graft_entry__
    __graft_entry__.build()
    from zigma_b200 import _lib
    return _lib


def test_ctypes_struct_layout_matches_c():
    _lib = _built()
    structs = {"zg_xattn_params": _lib.XattnParams, "zg_xattn_bwd_params": _lib.XattnBwdParams}
    lines = ['#include <stdio.h>', '#include <stddef.h>', f'#include "{HEADER}"', "int main(void) {"]
    for cname, st in structs.items():
        lines.append(f'printf("{cname} %zu\\n", sizeof({cname}));')
        for fname, _ in st._fields_:
            lines.append(f'printf("{cname}.{fname} %zu\\n", offsetof({cname}, {fname}));')
    lines.append("return 0; }")
    with tempfile.TemporaryDirectory() as d:
        src, exe = os.path.join(d, "l.c"), os.path.join(d, "l")
        open(src, "w").write("\n".join(lines))
        subprocess.check_call(["gcc", "-o", exe, src])
        out = subprocess.check_output([exe]).decode().split("\n")
    c_layout = dict(l.split() for l in out if l)
    for cname, st in structs.items():
        assert int(c_layout[cname]) == ctypes.sizeof(st), cname
        for fname, _ in st._fields_:
            assert int(c_layout[f"{cname}.{fname}"]) == getattr(st, fname).offset, f"{cname}.{fname}"


def test_abi_version_unchanged_and_exports():
    _lib = _built()
    assert _lib.lib().zg_abi_version() == 5
    for n in ("zg_cross_attn_fwd", "zg_cross_attn_bwd", "zg_cross_attn_bwd_workspace_bytes"):
        assert n in _lib.EXPORTS and hasattr(_lib.lib(), n)


def _fwd(_lib, p, batch, L, Lk, heads, dtype, esz, dim=None, offs=None, rs=None):
    """Fills params of contiguous (batch, L | Lk, dim) tensors at fake, 16-byte aligned addresses."""
    dim = heads * 64 if dim is None else dim
    rs = dim if rs is None else rs
    offs = offs or {}
    for i, n in enumerate(("q", "k", "v", "o")):
        setattr(p, n, FAKE * (i + 1) + offs.get(n, 0))
    p.lse = FAKE * 8
    for n in ("q", "o"):
        setattr(p, n + "_sb", L * rs); setattr(p, n + "_rs", rs)
    for n in ("k", "v"):
        setattr(p, n + "_sb", Lk * rs); setattr(p, n + "_rs", rs)
    p.batch, p.L, p.Lk, p.heads, p.dim, p.dtype = batch, L, Lk, heads, dim, dtype
    return p


def _bwd(_lib, batch, L, Lk, heads, dtype=None, sms=132, **kw):
    dtype = _lib.ZG_BF16 if dtype is None else dtype
    q = _lib.XattnBwdParams()
    _fwd(_lib, q.fwd, batch, L, Lk, heads, dtype, 2 if dtype else 4, **kw)
    dim = q.fwd.dim
    q.dout, q.dq, q.dk, q.dv = FAKE * 16, FAKE * 17, FAKE * 18, FAKE * 19
    q.dout_sb, q.dout_rs, q.dq_sb, q.dq_rs = L * dim, dim, L * dim, dim
    q.dk_sb, q.dk_rs, q.dv_sb, q.dv_rs = Lk * dim, dim, Lk * dim, dim
    q.sms = sms
    return q


def documented_workspace_bytes(B, L, Lk, H, sms):
    """The segment rule of include/zigma_b200.h, restated."""
    if B == 0 or L == 0:
        return 0
    cdiv = lambda a, b: -(-a // b)
    tiles = cdiv(L, 64)
    ctas = B * H * cdiv(Lk, 32)
    n = min(tiles, cdiv(8 * sms, ctas))
    per = cdiv(tiles, n)
    nseg = cdiv(tiles, per)
    return cdiv(4 * B * H * L, 16) * 16 + 2 * 4 * nseg * B * H * Lk * 64


def test_workspace_bytes_follow_the_segment_rule():
    _lib = _built()
    l = _lib.lib()
    for sms in (1, 78, 132, 148):
        for B in (0, 1, 2, 16, 64):
            for L in (0, 1, 37, 64, 65, 1024, 4096):
                for Lk in (1, 7, 77, 256):
                    for H in (1, 8):
                        q = _bwd(_lib, B, L, Lk, H, sms=sms)
                        assert l.zg_cross_attn_bwd_workspace_bytes(ctypes.byref(q)) == documented_workspace_bytes(B, L, Lk, H, sms), \
                            (B, L, Lk, H, sms)
    # the training shape of the demo model (bs 16, 1024 tokens, 8 heads, 77 keys) on a 132-SM H100: 3 segments of 384 rows
    assert documented_workspace_bytes(16, 1024, 77, 8, 132) == 16 * 8 * 1024 * 4 + 2 * 4 * 3 * 16 * 8 * 77 * 64 == 15_663_104


def _rc(_lib, name, q, ws_bytes=1 << 40):
    l = _lib.lib()
    if name == "fwd":
        return l.zg_cross_attn_fwd(ctypes.byref(q), ctypes.c_void_p(None))
    return l.zg_cross_attn_bwd(ctypes.byref(q), ctypes.c_void_p(FAKE * 64), ctypes.c_int64(ws_bytes), ctypes.c_void_p(None))


def test_argument_checks_on_empty_batches():
    """Accepted: B = 0 or L = 0 with any valid layout (nothing launched).  Rejected with an error, forward and backward: Lk
    outside [1, 256], an inner width that is not a multiple of 64 (or not 64 x heads), a pointer or stride off the 16-byte
    grid of the vector loads, and (backward) a workspace one byte short."""
    _lib = _built()
    l = _lib.lib()
    for dt, esz in ((_lib.ZG_F32, 4), (_lib.ZG_F16, 2), (_lib.ZG_BF16, 2)):
        for B, L in ((0, 64), (2, 0)):
            ok_f = _fwd(_lib, _lib.XattnParams(), B, L, 77, 8, dt, esz)
            assert _rc(_lib, "fwd", ok_f) == 0, l.zg_last_error()
            assert _rc(_lib, "bwd", _bwd(_lib, B, L, 77, 8, dt)) == 0, l.zg_last_error()
            assert _rc(_lib, "fwd", _fwd(_lib, _lib.XattnParams(), B, L, 1, 8, dt, esz)) == 0
            assert _rc(_lib, "fwd", _fwd(_lib, _lib.XattnParams(), B, L, 256, 1, dt, esz)) == 0
            # column slices of a fused (rows, 3 * 512) buffer: row stride 1536, offsets of 512 elements
            assert _rc(_lib, "fwd", _fwd(_lib, _lib.XattnParams(), B, L, 77, 8, dt, esz, rs=1536, offs={"k": 1024 * esz})) == 0
            for Lk in (0, 257, -1):
                assert _rc(_lib, "fwd", _fwd(_lib, _lib.XattnParams(), B, L, Lk, 8, dt, esz)) != 0 and b"Lk" in l.zg_last_error()
                assert _rc(_lib, "bwd", _bwd(_lib, B, L, Lk, 8, dt)) != 0 and b"Lk" in l.zg_last_error()
            for dim in (500, 520, 448):
                assert _rc(_lib, "fwd", _fwd(_lib, _lib.XattnParams(), B, L, 77, 8, dt, esz, dim=dim)) != 0
                assert b"inner width" in l.zg_last_error()
                assert _rc(_lib, "bwd", _bwd(_lib, B, L, 77, 8, dt, dim=dim)) != 0
            for n in ("q", "k", "v", "o"):
                off = 2 if esz == 2 else 4
                assert _rc(_lib, "fwd", _fwd(_lib, _lib.XattnParams(), B, L, 77, 8, dt, esz, offs={n: off})) != 0, n
                assert b"aligned" in l.zg_last_error()
                assert _rc(_lib, "bwd", _bwd(_lib, B, L, 77, 8, dt, offs={n: off})) != 0 and b"aligned" in l.zg_last_error()
            bad_rs = 512 + (4 if esz == 2 else 2)       # rows not on whole 16 bytes
            assert _rc(_lib, "fwd", _fwd(_lib, _lib.XattnParams(), B, L, 77, 8, dt, esz, rs=bad_rs)) != 0
            assert b"aligned" in l.zg_last_error()
            for n in ("dout", "dq", "dk", "dv"):
                q = _bwd(_lib, B, L, 77, 8, dt)
                setattr(q, n, getattr(q, n) + 2)
                assert _rc(_lib, "bwd", q) != 0 and b"aligned" in l.zg_last_error(), n
    # workspace: a non-empty call one byte short is rejected before any launch
    q = _bwd(_lib, 16, 1024, 77, 8)
    need = l.zg_cross_attn_bwd_workspace_bytes(ctypes.byref(q))
    assert _rc(_lib, "bwd", q, ws_bytes=need - 1) != 0 and b"workspace" in l.zg_last_error()
    q.sms = 0
    assert _rc(_lib, "bwd", q, ws_bytes=need) != 0 and b"sms" in l.zg_last_error()


XATTN_KERNELS = ["xattn_fwd_mma_kernel", "xattn_rows_kernel", "xattn_bwd_kv_kernel", "xattn_bwd_reduce_kernel"]


def test_sass_xattn_kernels_have_no_float_atomics():
    """Every instantiation: forward (tensor-core fp16 / bf16, CUDA-core fp32), backward dQ, dK / dV and segment reduction in
    three dtypes -- 12 functions, none with a floating-point RED / ATOM."""
    cuobjdump, filt = _tool("cuobjdump"), _tool("cu++filt")
    if cuobjdump is None or filt is None:
        pytest.skip("cuobjdump / cu++filt not available")
    _lib = _built()
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
    found = set()
    for mangled, dem in zip(names, demangled):
        m = re.search(r"zg::(xattn_\w+)<(.*)>\(", dem)
        if m is None:
            continue
        found.add((m.group(1), m.group(2).replace(" ", "")))
        bad = [l.strip() for l in funcs[mangled] if FLOAT_ATOMIC.search(l)]
        assert not bad, f"{dem}: {bad[:3]}"
    want = {("xattn_fwd_mma_kernel", t) for t in ("__half", "__nv_bfloat16")} | {("xattn_rows_kernel", "float,false")}
    want |= {(k, t + s) for k, s in (("xattn_rows_kernel", ",true"), ("xattn_bwd_kv_kernel", ""), ("xattn_bwd_reduce_kernel", ""))
             for t in ("float", "__half", "__nv_bfloat16")}
    norm = {(k, t.replace("(bool)1", "true").replace("(bool)0", "false")) for k, t in found}
    assert want <= norm, sorted(want - norm)
    assert len(want) == 12
    # the pattern does catch a floating-point atomic (the audit is not vacuous): the atomic scan backward has them
    atomic = [n for n, d in zip(names, demangled) if re.search(r"zg::scan_bwd_q4_kernel<.*, (?:false|\(bool\)0)>\(", d)]
    assert atomic and any(FLOAT_ATOMIC.search(l) for l in funcs[atomic[0]])
