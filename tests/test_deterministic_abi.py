"""CPU: the deterministic backward entry points (zg_*_bwd_det) -- workspace sizes at the BASELINE config-2 training shapes,
the too-small-workspace error, and a SASS audit of the built library: every DET kernel instantiation exists and none of
them contains a floating-point atomic or reduction.  No kernel is launched here (the size queries and the argument
checks are host code)."""
import ctypes as C
import os
import re
import shutil
import subprocess

import pytest

# config 2 (BASELINE.md: 32x32 latents, patch 1 -> L 1024, D 640, E 1280, dstate 16) at training batch 16
BS, L, D, E, N = 16, 1024, 640, 1280, 16
F32 = 4
FAKE = 1 << 20            # stands in for device pointers: the queries read addresses (alignment) only, never memory


def _built():
    import __graft_entry__
    __graft_entry__.build()
    from zigma_b200 import _lib
    return _lib


def _ptrs(obj, names, base=FAKE):
    for i, n in enumerate(names):
        setattr(obj, n, base * (i + 1))


def _scan_params(_lib, batch=BS, dim=E, seqlen=L, dstate=N, ngroups=1, var_bc=True, token_major=True):
    q = _lib.ScanBwdParams()
    p = q.fwd
    _ptrs(p, ["u", "delta", "z", "A", "D", "delta_bias", "ckpt"] + (["B", "C"] if var_bc else []))
    if not var_bc:
        p.B, p.C = FAKE * 20, FAKE * 21
    _ptrs(q, ["dout", "du", "ddelta", "dz", "dA", "dD", "ddelta_bias", "dB", "dC"], base=FAKE * 32)
    if token_major:
        for pre in ("u", "delta", "z"):
            setattr(p, pre + "_sb", seqlen * dim); setattr(p, pre + "_sd", 1); setattr(p, pre + "_sl", dim)
        for pre in ("dout", "du", "ddelta", "dz"):
            setattr(q, pre + "_sb", seqlen * dim); setattr(q, pre + "_sd", 1); setattr(q, pre + "_sl", dim)
        if var_bc:
            p.B_sb = p.C_sb = seqlen * ngroups * dstate
            p.B_sg = p.C_sg = dstate
            p.B_sn = p.C_sn = 1
            p.B_sl = p.C_sl = ngroups * dstate
    else:
        for pre in ("u", "delta", "z"):
            setattr(p, pre + "_sb", seqlen * dim); setattr(p, pre + "_sd", seqlen); setattr(p, pre + "_sl", 1)
        for pre in ("dout", "du", "ddelta", "dz"):
            setattr(q, pre + "_sb", seqlen * dim); setattr(q, pre + "_sd", seqlen); setattr(q, pre + "_sl", 1)
        if var_bc:
            p.B_sb = p.C_sb = ngroups * dstate * seqlen
            p.B_sg = p.C_sg = dstate * seqlen
            p.B_sn = p.C_sn = seqlen
            p.B_sl = p.C_sl = 1
    p.batch, p.dim, p.seqlen, p.dstate, p.ngroups = batch, dim, seqlen, dstate, ngroups
    p.dtype, p.ckpt_every = _lib.ZG_BF16, 8
    p.flags = _lib.SCAN_DELTA_SOFTPLUS | ((_lib.SCAN_VARIABLE_B | _lib.SCAN_VARIABLE_C) if var_bc else 0)
    return q


def _conv_params(_lib, token_major=True, bias=True):
    q = _lib.ConvBwdParams()
    p = q.fwd
    _ptrs(p, ["x", "weight", "out"])
    p.bias = FAKE * 8 if bias else None
    q.dout, q.dx, q.dweight = FAKE * 9, FAKE * 10, FAKE * 11
    q.dbias = FAKE * 12 if bias else None
    if token_major:       # x is the conv half of in_proj's (B, L, 2E) output: row stride 2E
        p.x_sb, p.x_sd, p.x_sl = L * 2 * E, 1, 2 * E
        q.dout_sb, q.dout_sd, q.dout_sl = L * E, 1, E
        q.dx_sb, q.dx_sd, q.dx_sl = L * 2 * E, 1, 2 * E
    else:
        p.x_sb, p.x_sd, p.x_sl = E * L, L, 1
        q.dout_sb, q.dout_sd, q.dout_sl = E * L, L, 1
        q.dx_sb, q.dx_sd, q.dx_sl = E * L, L, 1
    p.out_sb, p.out_sd, p.out_sl = q.dx_sb, q.dx_sd, q.dx_sl
    p.batch, p.dim, p.seqlen, p.width = BS, E, L, 4
    p.dtype, p.wdtype, p.silu = _lib.ZG_BF16, _lib.ZG_F32, 1
    return q


def _norm_params(_lib, ncols=D, bias=False):
    p = _lib.NormBwdParams()
    _ptrs(p, ["dy", "x", "weight", "rstd", "dx", "dweight"])
    p.dbias = FAKE * 16 if bias else None
    p.dy_rs = p.x_rs = p.dx_rs = ncols
    p.nrows, p.ncols = BS * L, ncols
    p.dtype, p.res_dtype, p.wdtype, p.is_rms = _lib.ZG_BF16, _lib.ZG_F32, _lib.ZG_F32, int(not bias)
    return p


def _tail_params(_lib, nparts, first=False):
    p = _lib.BlockTailBwdParams()
    _ptrs(p, ["d_residual_out", "d_modded", "r", "rstd", "scale", "norm_w", "d_x", "d_residual_in", "dshift", "dscale", "d_norm_w"])
    if not first:
        _ptrs(p, ["mix", "gate", "rowmap", "d_mix", "dgate"], base=FAKE * 64)
    p.mod_rs = 3 * D
    p.batch, p.seqlen, p.dim, p.dtype, p.nparts = BS, L, D, _lib.ZG_BF16, nparts
    return p


def test_abi_version_and_det_exports():
    _lib = _built()
    assert _lib.lib().zg_abi_version() == 5
    for op in _lib.DET_OPS:
        assert op + "_det" in _lib.EXPORTS and op + "_det_workspace_bytes" in _lib.EXPORTS


def test_scan_workspace_bytes():
    """dstate-16 kernel: dB / dC one row per 64-channel tile of the group (E / 64 = 20 rows of (batch, groups, 16, L) each:
    ~42 MB at config 2, bs 16), dA / dD / d(delta_bias) one row per batch row.  Generic kernel: two rows (warps) per tile for
    variable dB / dC, batch rows for constant ones."""
    _lib = _built()
    q = _scan_params(_lib)
    tiles = E // 64
    want = tiles * BS * 1 * N * L * F32 * 2 + BS * E * N * F32 + 2 * BS * E * F32
    assert want == 43_417_600
    assert _lib.det_workspace_bytes("zg_selective_scan_bwd", q) == want
    assert _lib.det_workspace_bytes("zg_selective_scan_bwd", _scan_params(_lib, token_major=False)) == want    # staged channel-first
    q.dD = None
    assert _lib.det_workspace_bytes("zg_selective_scan_bwd", q) == want - BS * E * F32
    # two groups: the tiles of one group
    q2 = _scan_params(_lib, ngroups=2)
    assert _lib.det_workspace_bytes("zg_selective_scan_bwd", q2) == (E // 2 // 64) * BS * 2 * N * L * F32 * 2 + BS * E * N * F32 + 2 * BS * E * F32
    # generic kernel, dstate 8, variable B / C: 2 warps per tile
    g8 = _scan_params(_lib, dim=256, seqlen=200, dstate=8, token_major=False)
    assert _lib.det_workspace_bytes("zg_selective_scan_bwd", g8) == (2 * 4) * BS * 8 * 200 * F32 * 2 + BS * 256 * 8 * F32 + 2 * BS * 256 * F32
    # generic kernel, constant B / C (dim, dstate): per batch row
    gc = _scan_params(_lib, dim=256, seqlen=200, dstate=16, var_bc=False, token_major=False)
    assert _lib.det_workspace_bytes("zg_selective_scan_bwd", gc) == 3 * BS * 256 * 16 * F32 + 2 * BS * 256 * F32
    # a misaligned A sends the dstate-16 call to the generic kernel: the layout follows
    q.dD = FAKE * 5
    q.fwd.A = FAKE * 4 + 4
    assert _lib.det_workspace_bytes("zg_selective_scan_bwd", q) == 2 * tiles * BS * N * L * F32 * 2 + BS * E * N * F32 + 2 * BS * E * F32


def test_conv_workspace_bytes():
    """Token-major fast kernel: one row per 4 (batch, 32-position chunk) rows; channel-first: one row per batch row."""
    _lib = _built()
    rows = (BS * (L // 32) + 3) // 4
    assert _lib.det_workspace_bytes("zg_causal_conv1d_bwd", _conv_params(_lib)) == rows * E * 5 * F32 == 3_276_800
    assert _lib.det_workspace_bytes("zg_causal_conv1d_bwd", _conv_params(_lib, bias=False)) == rows * E * 4 * F32
    assert _lib.det_workspace_bytes("zg_causal_conv1d_bwd", _conv_params(_lib, token_major=False)) == BS * E * 5 * F32
    q = _conv_params(_lib)
    q.fwd.dtype = _lib.ZG_F32                    # fp32 token-major: the generic kernel, 64-position chunks
    assert _lib.det_workspace_bytes("zg_causal_conv1d_bwd", q) == ((BS * (L // 64) + 3) // 4) * E * 5 * F32


def test_norm_and_tail_workspace_bytes():
    """add_norm: one row per CTA (vectorised) or warp (scalar) of the grid, capped at 528 CTAs whatever the device;
    block tail: (4 nparts / batch) warp rows of (batch, dim) per reduced output."""
    _lib = _built()
    assert _lib.det_workspace_bytes("zg_add_norm_bwd", _norm_params(_lib)) == 528 * D * F32
    assert _lib.det_workspace_bytes("zg_add_norm_bwd", _norm_params(_lib, bias=True)) == 2 * 528 * D * F32
    assert _lib.det_workspace_bytes("zg_add_norm_bwd", _norm_params(_lib, ncols=1280)) == 4 * 528 * 1280 * F32
    nparts = min((BS * L + 63) // 64, 3 * 132)   # block_ops' choice on a 132-SM H100
    wpb = 4 * nparts // BS
    assert _lib.det_workspace_bytes("zg_block_tail_bwd", _tail_params(_lib, nparts)) == 3 * wpb * BS * D * F32 == 7_864_320
    assert _lib.det_workspace_bytes("zg_block_tail_bwd", _tail_params(_lib, nparts, first=True)) == 2 * wpb * BS * D * F32


def test_det_call_rejects_small_workspace():
    """A workspace one byte short is an error returned before anything is launched (no GPU needed to see it)."""
    _lib = _built()
    l = _lib.lib()
    for name, q in (("zg_selective_scan_bwd", _scan_params(_lib)), ("zg_causal_conv1d_bwd", _conv_params(_lib)),
                    ("zg_add_norm_bwd", _norm_params(_lib)), ("zg_block_tail_bwd", _tail_params(_lib, 256))):
        need = _lib.det_workspace_bytes(name, q)
        rc = getattr(l, name + "_det")(C.byref(q), C.c_void_p(FAKE * 100), C.c_int64(need - 1), C.c_void_p(None))
        assert rc != 0 and b"workspace" in l.zg_last_error(), name
    q = _tail_params(_lib, 3)                    # 12 warps cannot give each of 16 batch elements its own
    rc = l.zg_block_tail_bwd_det(C.byref(q), C.c_void_p(FAKE * 100), C.c_int64(1 << 40), C.c_void_p(None))
    assert rc != 0 and b"nparts" in l.zg_last_error()


def test_tail_bwd_nparts_gives_every_batch_element_a_warp():
    """block_ops.tail_bwd_nparts, the CTA count of both block-tail backward kernels: at least one warp per batch element
    (small seqlen with a large batch, or a batch past 4 x 3 CTAs per SM), never more CTAs than the kernel accepts, and a
    batch beyond that a clear error rather than a failed launch."""
    from zigma_b200.block_ops import tail_bwd_nparts
    for sms in (1, 78, 114, 132, 148):
        for B in (1, 2, 3, 4, 5, 8, 9, 16, 64, 1584, 1585, 1600, 4096, 65535, 262140):
            for L in (1, 4, 5, 15, 16, 37, 256, 1024, 4096):
                n = tail_bwd_nparts(B, L, sms)
                assert 1 <= n <= 65535 and 4 * n >= B, (B, L, sms, n)
                assert n == max(1, min((B * L + 63) // 64, 3 * sms), (B + 3) // 4)
    assert tail_bwd_nparts(8, 4, 132) == 2 and tail_bwd_nparts(16, 1024, 132) == 256
    with pytest.raises(RuntimeError, match="65535"):
        tail_bwd_nparts(262141, 1, 132)


def _tail_fwd_params(_lib, dtype, dim, gate_off=0, scale_off=0):
    """Forward params of an EMPTY batch whose modulation vectors are views of one (batch, 3 dim) buffer at fake addresses: the
    argument checks run before the empty-batch return, so no kernel can be launched whatever they decide."""
    esz = 4 if dtype == _lib.ZG_F32 else 2
    p = _lib.BlockTailParams()
    _ptrs(p, ["x", "mix", "norm_w", "residual", "residual_out", "normed", "modded"])
    base = FAKE * 64
    p.gate, p.shift, p.scale = base + gate_off, base + dim * esz, base + 2 * dim * esz + scale_off
    p.mod_rs = 3 * dim
    p.batch, p.seqlen, p.dim, p.dtype = 0, 16, dim, dtype
    return p


def test_tail_modulation_alignment_checks():
    """zg_block_tail_fwd / _fwd_pe / _bwd read gate / shift / scale / norm_w as 4-element vectors: a pointer 2 bytes off is
    rejected by all three, while the views of a (batch, 3 dim) 16-bit buffer at dim = 36 (scale 144 bytes in, 8-byte
    aligned only) are accepted, forward and backward."""
    _lib = _built()
    l = _lib.lib()

    def fwd(name, p):
        if name == "zg_block_tail_fwd_pe":
            p.gate = p.residual = None
        return getattr(l, name)(C.byref(p), C.c_void_p(None))

    def bwd(p):
        q = _lib.BlockTailBwdParams()
        _ptrs(q, ["d_residual_out", "d_normed", "d_modded", "r", "rstd", "mix", "d_x", "d_mix", "d_residual_in",
                  "dgate", "dshift", "dscale", "d_norm_w"])
        q.gate, q.scale, q.norm_w = p.gate, p.scale, p.norm_w
        q.mod_rs, q.batch, q.seqlen, q.dim, q.dtype, q.nparts = p.mod_rs, 0, p.seqlen, p.dim, p.dtype, 1
        return l.zg_block_tail_bwd(C.byref(q), C.c_void_p(None))

    for dt in (_lib.ZG_F32, _lib.ZG_F16, _lib.ZG_BF16):
        for dim in (36, 100, 640):
            for name in ("zg_block_tail_fwd", "zg_block_tail_fwd_pe"):
                assert fwd(name, _tail_fwd_params(_lib, dt, dim)) == 0, (name, dt, dim, l.zg_last_error())
            assert bwd(_tail_fwd_params(_lib, dt, dim)) == 0, (dt, dim, l.zg_last_error())
            for off in ("gate_off", "scale_off"):
                p = _tail_fwd_params(_lib, dt, dim, **{off: 2})
                for name in ("zg_block_tail_fwd", "zg_block_tail_fwd_pe"):
                    if name == "zg_block_tail_fwd_pe" and off == "gate_off":
                        continue                   # the positional-embedding tail takes no gate
                    assert fwd(name, _tail_fwd_params(_lib, dt, dim, **{off: 2})) != 0, (name, off, dt, dim)
                    assert b"aligned" in l.zg_last_error()
                assert bwd(p) != 0 and b"aligned" in l.zg_last_error(), (off, dt, dim)
        p = _tail_fwd_params(_lib, dt, 64)
        p.norm_w += 2
        assert fwd("zg_block_tail_fwd", p) != 0 and bwd(p) != 0 and b"aligned" in l.zg_last_error()
    # fp32 needs 16 bytes: 8 bytes off, enough for a 16-bit vector, is rejected
    p = _tail_fwd_params(_lib, _lib.ZG_F32, 36, scale_off=8)
    assert fwd("zg_block_tail_fwd", p) != 0 and bwd(p) != 0


# kernel families with a DET instantiation (DET is the last template argument of each)
DET_KERNELS = ["scan_bwd_q4_kernel", "scan_bwd_kernel", "conv_bwd_seqc_kernel", "conv_bwd_seqc_vec_kernel", "conv_bwd_tok_kernel",
               "conv_bwd_tok4_kernel", "add_norm_bwd_kernel", "add_norm_bwd_vec_kernel", "block_tail_bwd_kernel"]
# an atomic or reduction (global or shared) with a floating-point add: REDG.E.ADD.F32.FTZ.RN.STRONG.GPU, ATOMS.ADD.F16x2, ...
FLOAT_ATOMIC = re.compile(r"\b(?:RED|ATOM)[A-Z]*(?:\.[A-Z0-9_]+)*\.ADD\.(?:F32|F16x2|BF16x2|F64)\b", re.IGNORECASE)


def _tool(name):
    return shutil.which(name) or (os.path.join("/usr/local/cuda/bin", name) if os.path.exists(os.path.join("/usr/local/cuda/bin", name)) else None)


def test_sass_det_kernels_have_no_float_atomics():
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
    assert len(demangled) == len(names)
    found = {k: 0 for k in DET_KERNELS}
    audited = 0
    for mangled, dem in zip(names, demangled):
        m = re.search(r"zg::(\w+)(?:<(.*)>)?\(", dem)
        if m is None or not (m.group(1) in DET_KERNELS or m.group(1) == "reduce_rows_kernel"):
            continue
        if m.group(1) != "reduce_rows_kernel":
            if m.group(2).split(",")[-1].strip() not in ("true", "(bool)1"):
                continue          # the atomic instantiation
            found[m.group(1)] += 1
        bad = [l.strip() for l in funcs[mangled] if FLOAT_ATOMIC.search(l)]
        assert not bad, f"{dem}: {bad[:3]}"
        audited += 1
    assert all(found.values()), f"DET instantiations missing: {[k for k, v in found.items() if not v]}"
    # and the pattern does catch the atomic twins (the audit is not vacuous)
    atomic = [n for n, d in zip(names, demangled) if re.search(r"zg::scan_bwd_q4_kernel<.*, (?:false|\(bool\)0)>\(", d)]
    assert atomic and any(FLOAT_ATOMIC.search(l) for l in funcs[atomic[0]])
    assert audited >= len(DET_KERNELS)
