"""GPU (H100): every instantiation of the add+norm and block-tail kernels of zigma_b200/csrc/norm.cu against a plain fp64
restatement of the same operation, at the model-zoo widths, in fp32 / fp16 / bf16, with and without
torch.use_deterministic_algorithms.

The references take exactly the values the kernels read (inputs are drawn in the kernel's dtype and upcast) and round to the
16-bit dtype where the kernels document a rounding point.  Bounds, instead of a blanket rtol:
* 16-bit outputs: distance in ulps of the dtype at the reference value, at most 1 (one rounding) or 2 (a chain of roundings),
  or, for an element formed by cancellation, the fp32 bound below plus one ulp; and the fraction of elements that differ
  from the rounded reference at all stays below MISMATCH[dtype] (a missing or extra rounding point moves tens of percent);
* fp32 elementwise outputs: |a - e| <= C_F32 * 2^-24 * M, M = the magnitude of the terms that form the element (never |e|,
  which is small exactly where the terms cancel);
* column sums (weight / bias / modulation gradients): |a - e| <= 1e-5 * S + one ulp of the returned dtype, S = sum of |term|
  over the summed rows; test_column_sum_bound_rejects_a_dropped_row shows that losing one row breaks it.
The achieved ulps, mismatch fractions and fp32 constants go to $ZIGMA_PARITY_LOG when it names a file."""
import re

import pytest
import torch

from util import COLSUM_REL, DTYPE_NAME, check_colsum, check_elem, ulp

DEV = "cuda"
gpu = pytest.mark.gpu

LOWP = (torch.float16, torch.bfloat16)
DTYPES = (torch.float32, torch.float16, torch.bfloat16)
_NAME = DTYPE_NAME


def test_column_sum_bound_rejects_a_dropped_row():
    """CPU: the column-sum bound passes a correctly rounded sum and rejects the same sum without any one row's contribution,
    at the row counts the matrix sums over and in every returned dtype (the bound is not vacuous)."""
    g = torch.Generator().manual_seed(0)
    for rows, cols in ((5003, 48), (1024, 64), (256, 36), (37, 640), (5, 368)):
        terms = torch.randn(rows, cols, generator=g, dtype=torch.float64) * torch.rand(rows, 1, generator=g, dtype=torch.float64).add(0.5)
        e, S = terms.sum(0), terms.abs().sum(0)
        for dt in DTYPES:
            check_colsum(f"selfcheck {rows}x{cols}", e.to(dt), e, S)
            for j in (0, rows // 2, rows - 1):
                dropped = (e - terms[j]).to(dt)
                bound = COLSUM_REL * S + ulp(e, dt)
                assert ((dropped.double() - e).abs() > bound).any(), (rows, cols, dt, j)
    # and the ulp bound of a 16-bit output rejects two ulps
    e = torch.randn(1000, generator=g, dtype=torch.float64)
    for dt in LOWP:
        check_elem("selfcheck ulp", e.to(dt), e, e.abs())
        with pytest.raises(AssertionError):
            check_elem("selfcheck 2 ulp", (e + 2 * ulp(e, dt)).to(dt), e, e.abs())


# ------------------------------------------------------------------------------------------------ add + norm
NORM_WIDTHS = (48, 368, 640, 768, 1024, 1028, 1536, 2048)     # vec MAXQ 2/4/5/6/8, then the scalar kernel
NORM_ROWS = (37, 1, 5003)          # 5003: every backward warp walks several rows (grid capped at 528 CTAs x 4 warps)


def _norm_cases():
    cases = []
    for N in NORM_WIDTHS:
        for T in DTYPES:
            for stream in (("none", "fp32", "T") if T in LOWP else ("none", "fp32")):
                cases.append((N, T, stream))
    return [c + (i,) for i, c in enumerate(cases)]


NORM_CASES = _norm_cases()


def _norm_setup(N, T, stream, i):
    """Inputs of one add+norm case.  The variant dimensions rotate with the case index i so that each meets every width,
    dtype and stream: RMS / LayerNorm with bias, weights in T or fp32 master weights, prenorm, row count, x / dy as column
    slices of wider tensors.  37-row cases carry edge rows: zeros, 1e-3 scale, one 1e3x outlier, and for fp32 LayerNorm
    a 1e3 common offset (which a one-pass E[x^2] - E[x]^2 would lose)."""
    g = torch.Generator().manual_seed(1000 + i)
    rn = lambda *s: torch.randn(*s, generator=g)
    rows = NORM_ROWS[i % 3]
    is_rms = i % 2 == 0
    prenorm = (i // 2) % 2 == 0
    wdt = torch.float32 if (T in LOWP and (i // 4) % 2 == 1) else T
    sliced = (i // 3) % 2 == 0
    has_res = stream == "T" or (stream == "fp32" and (i // 8) % 2 == 0)
    res_dt = T if stream == "T" else torch.float32
    x = rn(rows, N)
    res = rn(rows, N) if has_res else None
    if rows == 37:
        x[0] = 0
        x[1] *= 1e-3
        x[2, N // 3] *= 1e3
        if res is not None:
            res[0] = 0
            res[1] *= 1e-3
        if T == torch.float32 and not is_rms:
            x[3] += 1e3
    x = x.to(T)
    res = None if res is None else res.to(res_dt)
    w = (1 + 0.2 * rn(N)).to(wdt)
    b = None if is_rms else (0.2 * rn(N)).to(wdt)
    dy = rn(rows, N).to(T)
    dstream = rn(rows, N).to(res_dt if has_res else (torch.float32 if stream == "fp32" else T)) if prenorm else None
    return dict(x=x, res=res, w=w, b=b, dy=dy, dstream=dstream, is_rms=is_rms, prenorm=prenorm, sliced=sliced,
                fp32_stream=stream == "fp32", eps=1e-5 if i % 4 < 2 else 1e-6)


def _on_dev(t, sliced=False):
    """t on the GPU; sliced: as the leading columns of a wider tensor (row stride N + 4)."""
    if t is None:
        return None
    if not sliced:
        return t.to(DEV)
    wide = torch.zeros(t.shape[0], t.shape[1] + 4, dtype=t.dtype, device=DEV)
    wide[:, :t.shape[1]] = t.to(DEV)
    return wide[:, :t.shape[1]]


def ref_add_norm(c):
    """fp64 forward and backward of (residual add +) RMSNorm / LayerNorm.
    Forward: r = x + residual, statistics and y of the unrounded r, y rounded once to T; the stream is stored in its dtype.
    Backward: autograd of y = (r - mean) * rstd * w + b at the STORED stream r, with the forward's mean / rstd as values
    (the kernel saves them and reads the stored stream) and their derivatives 1/N and -rstd^3 (r - mean) / N."""
    x64 = c["x"].double()
    T = c["x"].dtype
    r_ex = x64 + (c["res"].double() if c["res"] is not None else 0)
    sdt = c["res"].dtype if c["res"] is not None else (torch.float32 if c["fp32_stream"] else None)
    r_st = r_ex.to(sdt).double() if sdt is not None else x64
    N = x64.shape[1]
    w = c["w"].double().requires_grad_()
    b = None if c["b"] is None else c["b"].double().requires_grad_()
    mean = torch.zeros(x64.shape[0], 1, dtype=torch.float64) if c["is_rms"] else r_ex.mean(-1, keepdim=True)
    rstd = ((r_ex - mean).pow(2).mean(-1, keepdim=True) + c["eps"]).rsqrt()
    y_fwd = (r_ex - mean) * rstd * w.detach() + (0 if b is None else b.detach())
    M_y = ((r_ex.abs() + mean.abs()) * rstd * w.detach().abs() + (0 if b is None else b.detach().abs()))

    r = r_st.clone().requires_grad_()
    mu = mean if c["is_rms"] else mean + (r.mean(-1, keepdim=True) - r.mean(-1, keepdim=True).detach())
    q = (r - mean).pow(2).mean(-1, keepdim=True) / 2
    rho = rstd - rstd.pow(3) * (q - q.detach())
    y = (r - mu) * rho * w + (0 if b is None else b)
    dy = c["dy"].double()
    loss = (y * dy).sum() + ((r * c["dstream"].double()).sum() if c["dstream"] is not None else 0)
    loss.backward()
    # magnitudes: xhat is formed from r and mean (a 1e3 offset row cancels there), c1 = mean(xhat * w dy), c2 = mean(w dy)
    xhat_mag = (r_st.abs() + mean.abs()) * rstd
    wdy = (dy * w.detach()).abs()
    M_dx = (wdy + xhat_mag * (xhat_mag * wdy).mean(-1, keepdim=True) + (0 if c["is_rms"] else wdy.mean(-1, keepdim=True))) * rstd
    if c["dstream"] is not None:
        M_dx = M_dx + c["dstream"].double().abs()
    out = dict(y=y_fwd, M_y=M_y, stream=r_ex if sdt is not None else None, sdt=sdt,
               M_stream=x64.abs() + (c["res"].double().abs() if c["res"] is not None else 0),
               dx=r.grad, M_dx=M_dx, dw=w.grad, S_dw=(dy.abs() * xhat_mag).sum(0))
    if b is not None:
        out.update(db=b.grad, S_db=dy.abs().sum(0))
    return out


def _run_add_norm(c):
    """The kernels through rms_norm_fn / layer_norm_fn and autograd; returns the outputs and the gradients."""
    from zigma_b200 import layer_norm_fn
    x = _on_dev(c["x"], c["sliced"]).requires_grad_()
    res = None if c["res"] is None else c["res"].to(DEV).requires_grad_()
    w = c["w"].to(DEV).requires_grad_()
    b = None if c["b"] is None else c["b"].to(DEV).requires_grad_()
    out = layer_norm_fn(x, w, b, residual=res, eps=c["eps"], prenorm=c["prenorm"], residual_in_fp32=c["fp32_stream"],
                        is_rms_norm=c["is_rms"])
    y, stream = out if c["prenorm"] else (out, None)
    dy = _on_dev(c["dy"], c["sliced"])
    if c["prenorm"]:
        torch.autograd.backward([y, stream], [dy, c["dstream"].to(DEV)])
    else:
        y.backward(dy)
    return dict(y=y, stream=stream, dx=x.grad, dres=None if res is None else res.grad, dw=w.grad, db=None if b is None else b.grad)


def _check_add_norm(tag, c, ref, got):
    T = c["x"].dtype
    check_elem(f"{tag} y", got["y"], ref["y"], ref["M_y"])
    if got["stream"] is not None and ref["sdt"] is not None:
        check_elem(f"{tag} residual_out", got["stream"], ref["stream"], ref["M_stream"])
    check_elem(f"{tag} dx", got["dx"], ref["dx"], ref["M_dx"])
    if got["dres"] is not None:
        assert got["dres"].dtype == c["res"].dtype
        check_elem(f"{tag} dresidual", got["dres"], ref["dx"], ref["M_dx"])
    check_colsum(f"{tag} dweight", got["dw"], ref["dw"], ref["S_dw"])
    if c["b"] is not None:
        check_colsum(f"{tag} dbias", got["db"], ref["db"], ref["S_db"])
    assert got["y"].dtype == T and got["dx"].dtype == T


def _add_norm_misaligned_dy(c):
    """_norm_bwd called directly with dy 8 bytes past a 16-byte boundary: the scalar kernel at a width the vector kernel has."""
    from zigma_b200.layernorm import _norm_fwd, _norm_bwd
    T = c["x"].dtype
    x, res = c["x"].to(DEV), None if c["res"] is None else c["res"].to(DEV)
    w, b = c["w"].to(DEV), None if c["b"] is None else c["b"].to(DEV)
    sdt = res.dtype if res is not None else (torch.float32 if c["fp32_stream"] else None)
    y, mean, rstd, stream = _norm_fwd(x, w, b, c["eps"], res, sdt, c["is_rms"])
    k = 8 // c["dy"].element_size()
    buf = torch.empty(c["dy"].numel() + k, dtype=T, device=DEV)
    dy = buf[k:].view(c["dy"].shape)
    dy.copy_(c["dy"].to(DEV))
    assert dy.data_ptr() % 16 == 8
    dst = None if c["dstream"] is None else c["dstream"].to(DEV).to(stream.dtype)
    dx, dw, db, dres = _norm_bwd(dy, stream, w, b, mean, rstd, dst, res is not None, c["is_rms"], T)
    return dict(y=y, stream=None, dx=dx, dres=dres if (res is not None and dres is not dx) else None, dw=dw, db=db)


@gpu
@pytest.mark.parametrize("N,T,stream,i", NORM_CASES, ids=[f"{n}-{_NAME[t]}-{s}" for n, t, s, _ in NORM_CASES])
def test_add_norm_vs_fp64(N, T, stream, i):
    c = _norm_setup(N, T, stream, i)
    ref = ref_add_norm(c)
    tag = f"add_norm {N} {_NAME[T]} stream={stream} rms={c['is_rms']} rows={c['x'].shape[0]} w={_NAME[c['w'].dtype]} prenorm={c['prenorm']}"
    for det in (False, True):
        with _deterministic(det):
            _check_add_norm(f"{tag} det={det}", c, ref, _run_add_norm(c))
            if N == 640:
                _check_add_norm(f"{tag} det={det} misaligned dy", c, ref, _add_norm_misaligned_dy(c))


class _deterministic:
    def __init__(self, on):
        self.on = on

    def __enter__(self):
        self.prev = torch.are_deterministic_algorithms_enabled()
        torch.use_deterministic_algorithms(self.on)

    def __exit__(self, *a):
        torch.use_deterministic_algorithms(self.prev)


# ------------------------------------------------------------------------------------------------ block tail forward
TAIL_FWD_WIDTHS = (36, 368, 640, 768, 1024, 1536, 2048)        # row4 kernel Q = 1, 1, 2, 2, 2, 3, 4
TAIL_VARIANTS = ("first", "middle", "middle_rowmap", "final", "pe")


def _rd(v, T):
    return v.to(T).double()


def _tail_inputs(B, L, D, T, seed, edge=True):
    """x, mix (B, L, D), residual (fp32), mods (B, 3D) as shift | scale | gate (adaLN's chunk order), norm_w, rowmap (a
    permutation).  Edge rows of batch element 0 (via the mix row they read): zeros, 1e-3 scale, one 1e3x outlier."""
    g = torch.Generator().manual_seed(seed)
    rn = lambda *s: torch.randn(*s, generator=g)
    x, mix, res = rn(B, L, D), rn(B, L, D), rn(B, L, D)
    perm = torch.randperm(L, generator=g)
    if edge and L >= 3:
        for l, s in ((0, 0.0), (1, 1e-3)):
            x[0, l] *= s
            res[0, l] *= s
            mix[0, perm[l]] *= s
        x[0, 2, D // 3] *= 1e3
    mods = (0.3 * rn(B, 3 * D)).to(T)
    nw = (1 + 0.2 * rn(D)).to(T)
    return x.to(T), mix.to(T), res, mods, nw, perm


def ref_tail_fwd(x, mix_rows, gate, nw, res, eps, final, T):
    """fp64 block tail forward with the kernel's rounding points (eager-torch order):
    h = round(x + round(gate * mix)); r = residual + h (fp32); normed = round(r * rstd * w);
    final: LayerNorm(no affine, 1e-6) of the rounded normed.  (modded: ref_modulate.)
    mix_rows: the mix row each token reads, already gathered; gate None with mix: the positional-embedding add (gate 1)."""
    h, M_h = x.double(), x.double().abs()
    if mix_rows is not None:
        gm = mix_rows.double() if gate is None else _rd(gate.double()[:, None] * mix_rows.double(), T)
        h = _rd(h + gm, T)
        M_h = M_h + gm.abs()
    r, M_r = (h + res.double(), M_h + res.double().abs()) if res is not None else (h, M_h)
    rstd = (r.pow(2).mean(-1, keepdim=True) + eps).rsqrt()
    n_pre = r * rstd * nw.double()
    M_n = M_r * rstd * nw.double().abs()
    out = dict(r=r, M_r=M_r, normed=n_pre, M_normed=M_n)
    if final:
        n = _rd(n_pre, T)
        mean = n.mean(-1, keepdim=True)
        rstd2 = ((n - mean).pow(2).mean(-1, keepdim=True) + 1e-6).rsqrt()
        out.update(normed=(n - mean) * rstd2, M_normed=(M_n + mean.abs()) * rstd2,
                   extra=ulp(n, T) * rstd2 if T in LOWP else None)
    return out


def ref_modulate(normed, shift, scale, T):
    """modded = round(round(normed * round(1 + scale)) + shift), from the normed output the kernel stored (and modulated)."""
    n = normed.detach().double().cpu()
    s1 = _rd(1 + scale.double()[:, None], T)
    return _rd(n * s1, T) + shift.double()[:, None], (n * s1).abs() + shift.double()[:, None].abs()


def _tail_fwd_case(T, D, variant, k, check=True):
    from zigma_b200.engine import block_tail
    B, L, eps = 3, 37, 1e-5
    x, mix, res, mods, nw, perm = _tail_inputs(B, L, D, T, seed=100 * D + k)
    views = k % 2 == 0                      # modulation as views of one (B, 3D) tensor, or as separate (B, D) tensors
    md = mods.to(DEV)
    dshift, dscale, dgate = (md[:, :D], md[:, D:2 * D], md[:, 2 * D:]) if views else \
        tuple(md[:, j * D:(j + 1) * D].clone() for j in range(3))
    shift, scale, gate = mods[:, :D], mods[:, D:2 * D], mods[:, 2 * D:]
    xd, mixd, resd, nwd = x.to(DEV), mix.to(DEV), res.to(DEV), nw.to(DEV)
    rowmap = perm.to(DEV).to(torch.int32) if variant in ("middle_rowmap", "final") else None
    src = perm if rowmap is not None else torch.arange(L)
    if variant == "first":
        got = block_tail(xd, None, None, dshift, dscale, nwd, None, None, eps)
        ref = None if not check else ref_tail_fwd(x, None, None, nw, None, eps, False, T)
    elif variant == "pe":
        pe = mix[0]
        got = block_tail(xd, pe.to(DEV), None, dshift, dscale, nwd, None, None, eps, mix_bcast=True)
        ref = None if not check else ref_tail_fwd(x, pe[None].expand(B, L, D), None, nw, None, eps, False, T)
    else:
        final = variant == "final"
        got = block_tail(xd, mixd, dgate, None if final else dshift, None if final else dscale, nwd, resd, rowmap, eps, final=final)
        ref = None if not check else ref_tail_fwd(x, mix[:, src], gate, nw, res, eps, final, T)
    if not check:
        return
    tag = f"tail fwd {_NAME[T]} D={D} {variant} {'views' if views else 'separate'}"
    r_out, normed, modded = got
    if r_out is not None:
        check_elem(f"{tag} residual_out", r_out, ref["r"], ref["M_r"])
    check_elem(f"{tag} normed", normed, ref["normed"], ref["M_normed"], max_ulp=2, extra=ref.get("extra"))
    if modded is not None:
        check_elem(f"{tag} modded", modded, *ref_modulate(normed, shift, scale, T), max_ulp=2)


@gpu
@pytest.mark.parametrize("D", TAIL_FWD_WIDTHS)
@pytest.mark.parametrize("T", DTYPES, ids=[_NAME[t] for t in DTYPES])
def test_block_tail_fwd_vs_fp64(T, D):
    for k, variant in enumerate(TAIL_VARIANTS):
        _tail_fwd_case(T, D, variant, k)


# ------------------------------------------------------------------------------------------------ block tail backward
TAIL_BWD_WIDTHS = (36, 368, 640, 768, 1024)                   # MAXQ 4, 4, 5, 6, 8
# (first block, absent output gradient, (B, L), rowmap): (3, 37) warp ranges straddle a batch boundary, (9, 5) one warp
# spans several batch elements, (4, 256) a config-2-like shape
TAIL_BWD_CONFIGS = ((False, None, (3, 37), True), (False, "d_residual_out", (9, 5), True), (True, "d_normed", (4, 256), False),
                    (False, "d_modded", (4, 256), False), (True, None, (9, 5), False))


def ref_tail_bwd(r, nw, shift_scale_gate, d_ro, d_n, d_m, eps, T):
    """fp64 autograd of r -> normed = r * rstd(r) * w, modded = normed * (1 + scale) + shift at the forward's saved fp32 r
    (unrounded 1 + scale: the backward's formula): dr (d_residual_in; d_x = dh = round(dr)) and the column sums but dgate.
    d_mix = round(gate * dh) and dgate = sum dh * mix follow from the kernel's own dh (its d_x output): ref_gated."""
    _, scale, _ = shift_scale_gate
    r = r.double().requires_grad_()
    w = nw.double().requires_grad_()
    sc = scale.double().requires_grad_()
    sh = torch.zeros_like(sc, requires_grad=True)
    rstd = (r.pow(2).mean(-1, keepdim=True) + eps).rsqrt()
    xh = r * rstd
    n = xh * w
    m = n * (1 + sc[:, None]) + sh[:, None]
    loss = sum((o * g_.double()).sum() for o, g_ in ((r, d_ro), (n, d_n), (m, d_m)) if g_ is not None)
    loss.backward()
    dr = r.grad
    dy_mag = (d_n.double().abs() if d_n is not None else 0) + (d_m.double().abs() * (1 + sc.detach()[:, None]).abs() if d_m is not None else 0)
    xh = xh.detach()
    wd = w.detach().abs()
    M_dr = (dy_mag * wd + xh.abs() * (xh.abs() * wd * dy_mag).mean(-1, keepdim=True)) * rstd.detach() + (d_ro.abs().double() if d_ro is not None else 0)
    zeros = torch.zeros_like(sc)
    out = dict(dr=dr, M_dr=M_dr, dh=_rd(dr, T), d_norm_w=w.grad, S_norm_w=(dy_mag * xh.abs()).sum((0, 1)),
               dshift=zeros if sh.grad is None else sh.grad, S_dshift=d_m.double().abs().sum(1) if d_m is not None else zeros,
               dscale=zeros if sc.grad is None else sc.grad, S_dscale=(d_m.double() * n.detach()).abs().sum(1) if d_m is not None else zeros)
    return out


def ref_gated(dh, gate, mix_rows):
    """d_mix = round(gate * dh) (token order) and dgate = sum_l dh * mix[rowmap[l]] from the dh = d_x the kernel stored."""
    dh = dh.detach().double().cpu()
    gm = gate.double()[:, None] * dh
    return gm, gm.abs(), (dh * mix_rows.double()).sum(1), (dh * mix_rows.double()).abs().sum(1)


def _tail_bwd_case(T, D, cfg, k, det, check=True, nw_master=False, edge=True):
    """block_tail_fn forward + backward for one configuration; checks every output and gradient against ref_tail_bwd."""
    from zigma_b200.block_ops import block_tail_fn
    first, absent, (B, L), use_rowmap = cfg
    eps = 1e-5
    x, mix, res, mods, nw, perm = _tail_inputs(B, L, D, T, seed=7 * D + 31 * k + 1, edge=edge)
    if nw_master:
        nw = nw.float()
    g = torch.Generator().manual_seed(5 * D + k)
    grads = {n_: torch.randn(B, L, D, generator=g).to(torch.float32 if n_ == "d_residual_out" else T)
             for n_ in ("d_residual_out", "d_normed", "d_modded") if n_ != absent}
    md = mods.to(DEV).requires_grad_()
    views = k % 2 == 0
    if views:
        dshift, dscale, dgate = md.chunk(3, dim=1)
    else:
        sep = [md.detach()[:, j * D:(j + 1) * D].clone().requires_grad_() for j in range(3)]
        dshift, dscale, dgate = sep
    xd, nwd = x.to(DEV).requires_grad_(), nw.to(DEV).requires_grad_()
    mixd, resd = (None, None) if first else (mix.to(DEV).requires_grad_(), res.to(DEV).requires_grad_())
    rowmap = perm.to(DEV).to(torch.int32) if (use_rowmap and not first) else None
    with _deterministic(det):
        r_out, normed, modded = block_tail_fn(xd, mixd, None if first else dgate, dshift, dscale, nwd, resd, rowmap, eps)
        outs = [(o, grads[n_].to(DEV)) for o, n_ in ((r_out, "d_residual_out"), (normed, "d_normed"), (modded, "d_modded")) if n_ in grads]
        torch.autograd.backward([o for o, _ in outs], [g_ for _, g_ in outs])
    if not check:
        return
    src = perm if (use_rowmap and not first) else torch.arange(L)
    shift, scale, gate = mods[:, :D], mods[:, D:2 * D], mods[:, 2 * D:]
    ref = ref_tail_bwd(r_out.detach().cpu(), nw.to(T), (shift, scale, gate),
                       grads.get("d_residual_out"), grads.get("d_normed"), grads.get("d_modded"), eps, T)
    tag = f"tail bwd {_NAME[T]} D={D} {B}x{L} first={first} absent={absent} rowmap={rowmap is not None} det={det}"
    check_elem(f"{tag} dx", xd.grad, ref["dr"], ref["M_dr"])
    if not first:
        check_elem(f"{tag} d_residual_in", resd.grad, ref["dr"], ref["M_dr"])
        e_mix, M_mix, e_gate, S_gate = ref_gated(xd.grad, gate, mix[:, src])
        d_mix = torch.empty_like(e_mix)
        d_mix[:, src] = e_mix                                         # back to the scan order the mixer produced
        M_d_mix = torch.empty_like(d_mix)
        M_d_mix[:, src] = M_mix
        check_elem(f"{tag} d_mix", mixd.grad, d_mix, M_d_mix, max_ulp=2)
    if views:
        dmods = md.grad
        got_sh, got_sc, got_g = dmods[:, :D], dmods[:, D:2 * D], dmods[:, 2 * D:]
    else:
        got_sh, got_sc, got_g = (t_.grad for t_ in sep)
    check_colsum(f"{tag} dshift", got_sh, ref["dshift"], ref["S_dshift"])
    check_colsum(f"{tag} dscale", got_sc, ref["dscale"], ref["S_dscale"])
    if first:
        assert got_g is None or not got_g.any()
    else:
        check_colsum(f"{tag} dgate", got_g, e_gate, S_gate)
    assert nwd.grad.dtype == nw.dtype
    check_colsum(f"{tag} d_norm_w", nwd.grad, ref["d_norm_w"], ref["S_norm_w"])


@gpu
@pytest.mark.parametrize("D", TAIL_BWD_WIDTHS)
@pytest.mark.parametrize("T", DTYPES, ids=[_NAME[t] for t in DTYPES])
def test_block_tail_bwd_vs_fp64(T, D):
    for k, cfg in enumerate(TAIL_BWD_CONFIGS):
        for det in (False, True):
            _tail_bwd_case(T, D, cfg, k, det, nw_master=(T in LOWP and k == 1))


@gpu
@pytest.mark.parametrize("T,B,L,D,dets", [(torch.bfloat16, 3, 37, 36, (False, True)), (torch.bfloat16, 3, 37, 100, (False, True)),
                                          (torch.float32, 8, 4, 64, (True,)), (torch.bfloat16, 8, 4, 64, (True,)),
                                          (torch.float32, 1600, 16, 64, (True,))],
                         ids=["bf16-D36", "bf16-D100", "det-8x4-fp32", "det-8x4-bf16", "det-1600x16"])
def test_block_tail_fn_shapes_that_failed(T, B, L, D, dets):
    """block_tail_fn forward + backward where it used to raise: 16-bit widths with D % 8 == 4 (the scale view of adaLN's
    (B, 3D) output is 8- but not 16-byte aligned), and the deterministic backward with fewer CTAs than batch elements / 4
    (small seqlen with batch > 4, batch > 1584)."""
    for det in dets:
        for k, (first, absent) in enumerate(((False, None), (True, "d_residual_out"))):
            _tail_bwd_case(T, D, (first, absent, (B, L), True), 2 * k, det, edge=False)


# ------------------------------------------------------------------------------------------------ coverage
# The dispatch tables of norm.cu, written out: (T, R) pairs of the add+norm kernels, the MAXQ buckets of the vectorised
# backward, the Q buckets of the four-warps-per-row tail forward (PE and not), the MAXQ buckets of the tail backward; DET
# (the last template argument) both ways.  Not listed: the one-warp-per-row block_tail_kernel, reached only with
# ZG_TAIL_ROW4=0 (read once per process) or 2^31 rows or more; whether to keep it is a separate question.
NORM_TR = (("float", "float"), ("__half", "float"), ("__half", "__half"), ("__nv_bfloat16", "float"), ("__nv_bfloat16", "__nv_bfloat16"))
TAIL_T = ("float", "__half", "__nv_bfloat16")
BOOLS = ("false", "true")
EXPECTED_KERNELS = (
    {("add_norm_fwd_kernel", (t, r)) for t, r in NORM_TR}
    | {("add_norm_bwd_vec_kernel", (t, r, str(q), d)) for t, r in NORM_TR for q in (2, 4, 5, 6, 8) for d in BOOLS}
    | {("add_norm_bwd_kernel", (t, r, d)) for t, r in NORM_TR for d in BOOLS}
    | {("block_tail_row4_kernel", (t, str(q), pe)) for t in TAIL_T for q in (1, 2, 3, 4) for pe in BOOLS}
    | {("block_tail_bwd_kernel", (t, str(q), d)) for t in TAIL_T for q in (4, 5, 6, 8) for d in BOOLS})
NORM_KERNELS = {"add_norm_fwd_kernel", "add_norm_bwd_vec_kernel", "add_norm_bwd_kernel", "block_tail_kernel", "block_tail_row4_kernel",
                "block_tail_bwd_kernel"}


def _template_args(s):
    out = []
    for a in s.split(","):
        a = a.strip()
        a = {"(bool)1": "true", "(bool)0": "false"}.get(a, a)
        out.append(re.sub(r"^\((?:int|unsigned int)\)", "", a))
    return tuple(out)


@gpu
def test_matrix_reaches_every_norm_kernel_instantiation():
    """The cases above, run once more without the reference under torch.profiler: the set of norm.cu kernels they launch is
    exactly the dispatch tables (5 + 50 + 10 + 24 + 24 instantiations)."""
    assert len(EXPECTED_KERNELS) == 113
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for N, T, stream, i in NORM_CASES:
            c = _norm_setup(N, T, stream, i)
            for det in (False, True):
                with _deterministic(det):
                    _run_add_norm(c)
                    if N == 640:
                        _add_norm_misaligned_dy(c)
        for T in DTYPES:
            for D in TAIL_FWD_WIDTHS:
                for k, variant in enumerate(TAIL_VARIANTS):
                    _tail_fwd_case(T, D, variant, k, check=False)
            for D in TAIL_BWD_WIDTHS:
                for k, cfg in enumerate(TAIL_BWD_CONFIGS):
                    for det in (False, True):
                        _tail_bwd_case(T, D, cfg, k, det, check=False)
        torch.cuda.synchronize()
    seen = set()
    for evt in prof.events():
        m = re.search(r"zg::(\w+)<(.*)>\(", evt.name)
        if m and m.group(1) in NORM_KERNELS:
            seen.add((m.group(1), _template_args(m.group(2))))
    assert seen, "the profiler recorded no norm.cu kernel"
    missing, extra = sorted(EXPECTED_KERNELS - seen), sorted(seen - EXPECTED_KERNELS)
    assert not missing and not extra, f"not launched: {missing}\nlaunched but not in the dispatch tables: {extra}"
