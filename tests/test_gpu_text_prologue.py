"""GPU (H100): the text prologue of has_text blocks (zg_text_prologue_fwd / _bwd, block_ops.TextPrologueFn, the fused
training loop and the sampling engine's text branch).

Kernels against an fp64 restatement of the formulas in include/zigma_b200.h, with the per-element bounds of
test_gpu_norm_kernels.py (util.check_elem / check_colsum).  The references take exactly the values the kernels read; where a
rounded intermediate is formed by fp32 operations that are exact or identical in both (ln = round((hidden - mean) * rstd)
from the saved fp32 statistics, the product of two 16-bit values), the reference recomputes it the same way, and the
statistics themselves are checked against fp64.  Models: the fused loop against the per-op block loop
(ZIGMA_FUSED_TRAIN_TAIL=0) at test_gpu_bwd.py's tolerances, and the profiler for what an engine forward and a training step
launch."""
import contextlib
import os

import pytest
import torch

from util import DTYPE_NAME, check_close, check_colsum, check_elem, model_case, ulp

DEV = "cuda"
gpu = pytest.mark.gpu
DTYPES = (torch.float32, torch.float16, torch.bfloat16)
LOWP = (torch.float16, torch.bfloat16)
EPS = 1e-6


@contextlib.contextmanager
def _deterministic(on):
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(on)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(prev)


def _rd(v, T):
    return v.to(T).double()


def _rowmap(kind, L, fold, g):
    """(int32 table or None, the mix row each token of a (B fold, L / fold) row reads)."""
    n = L // fold
    if kind == "none":
        return None, torch.arange(n)
    if kind == "zigzag":
        perm = torch.randperm(n, generator=g)
        return perm, perm
    # composite table of a copy-free temporal video layer: position k T + t of the (k, t) layout <-> token (perm[t], k)
    T = 4
    K = n // T
    perm = torch.randperm(T, generator=g)
    rev = torch.argsort(perm)
    k = torch.arange(K)
    comp_out = (k.view(1, K) * T + rev.view(T, 1)).reshape(-1)
    return comp_out, comp_out


def _inputs(B, L, D, T, fold, kind, seed):
    g = torch.Generator().manual_seed(seed)
    rn = lambda *s: torch.randn(*s, generator=g)
    Bf = B * fold
    x, mix = rn(Bf, L // fold, D), rn(Bf, L // fold, D)
    x[0, 0] *= 0.0
    if L // fold > 2:
        x[0, 1] *= 1e-3
        x[0, 2, D // 3] *= 1e2
    mods = (0.3 * rn(B, 6 * D)).to(T)            # adaLN's 6 chunks: gate, shift, scale of the text branch are 2, 3, 4
    table, src = _rowmap(kind, L, fold, g)
    return x.to(T), mix.to(T), mods, table, src


def _ln32(hidden, mean, rstd, T):
    """ln = round((hidden - mean) * rstd) with the kernel's fp32 operations on its saved statistics (bitwise the kernel's)."""
    h = hidden.detach().float().cpu()
    return _rd((h - mean.cpu().view(h.shape[:2] + (1,))) * rstd.cpu().view(h.shape[:2] + (1,)), T)


def _fwd_case(T, D, B, L, fold, kind, seed):
    from zigma_b200.engine import text_prologue
    x, mix, mods, table, src = _inputs(B, L, D, T, fold, kind, seed)
    md = mods.to(DEV)
    gate, shift, scale = md[:, 2 * D:3 * D], md[:, 3 * D:4 * D], md[:, 4 * D:5 * D]
    rowmap = None if table is None else table.to(torch.int32).to(DEV)
    hidden, q_in, mean, rstd = text_prologue(x.to(DEV), mix.to(DEV), gate, shift, scale, rowmap, EPS, mod_div=fold, want_stats=True)
    tag = f"text fwd {DTYPE_NAME[T]} D={D} {B}x{L} fold={fold} {kind}"
    per = lambda t: t.double().repeat_interleave(fold, dim=0)[:, None]     # per-row modulation of the (B fold) rows
    gm = _rd(per(mods[:, 2 * D:3 * D]) * mix[:, src].double(), T)
    check_elem(f"{tag} hidden", hidden, x.double() + gm, x.double().abs() + gm.abs())
    h = hidden.detach().double().cpu()
    e_mean = h.mean(-1)
    e_rstd = ((h - e_mean[..., None]).pow(2).mean(-1) + EPS).rsqrt()
    M_mean = h.abs().mean(-1)
    check_elem(f"{tag} mean", mean.view(h.shape[:2]), e_mean, M_mean)
    check_elem(f"{tag} rstd", rstd.view(h.shape[:2]), e_rstd, e_rstd * (1 + M_mean * e_rstd))
    ln = _ln32(hidden, mean, rstd, T)
    s1 = _rd(1 + per(mods[:, 4 * D:5 * D]), T)
    prod = _rd(ln * s1, T)
    sh = per(mods[:, 3 * D:4 * D])
    check_elem(f"{tag} q_in", q_in, prod + sh, prod.abs() + sh.abs())
    return hidden, q_in


FWD_WIDTHS = (64, 368, 768, 1024, 1536, 2048)       # Q 1, 1, 2, 2, 3, 4
# (B, L, fold, row table): ragged batch / seqlen, the zigzag table, the composite temporal table, a spatial video layer
FWD_CONFIGS = ((3, 37, 1, "none"), (2, 64, 1, "zigzag"), (2, 32, 1, "temporal"), (2, 64, 4, "zigzag"), (1, 1, 1, "none"))


@gpu
@pytest.mark.parametrize("D", FWD_WIDTHS)
@pytest.mark.parametrize("T", DTYPES, ids=[DTYPE_NAME[t] for t in DTYPES])
def test_forward_vs_fp64(T, D):
    for k, (B, L, fold, kind) in enumerate(FWD_CONFIGS):
        _fwd_case(T, D, B, L, fold, kind, seed=17 * D + k)


def _bwd_case(T, D, B, L, kind, det, seed, with_dh=True):
    from zigma_b200.block_ops import text_prologue_fn
    x, mix, mods, table, src = _inputs(B, L, D, T, 1, kind, seed)
    g = torch.Generator().manual_seed(seed + 5)
    d_hid = torch.randn(B, L, D, generator=g).to(T) if with_dh else None
    d_q = torch.randn(B, L, D, generator=g).to(T)
    md = mods.to(DEV).requires_grad_()
    chunks = md.chunk(6, dim=1)
    xd, mixd = x.to(DEV).requires_grad_(), mix.to(DEV).requires_grad_()
    rowmap = None if table is None else table.to(torch.int32).to(DEV)
    with _deterministic(det):
        hidden, q_in = text_prologue_fn(xd, mixd, chunks[2], rowmap, chunks[3], chunks[4], EPS)
        outs = [q_in] + ([hidden] if with_dh else [])
        torch.autograd.backward(outs, [d_q.to(DEV)] + ([d_hid.to(DEV)] if with_dh else []))
    tag = f"text bwd {DTYPE_NAME[T]} D={D} {B}x{L} {kind} d_hidden={with_dh} det={det}"
    # statistics as the kernel saved them (TextPrologueFn's forward ran the checked forward kernel)
    from zigma_b200.engine import text_prologue
    _, _, mean, rstd = text_prologue(xd.detach(), mixd.detach(), chunks[2].detach(), chunks[3].detach(), chunks[4].detach(), rowmap,
                                     EPS, want_stats=True)
    h = hidden.detach().double().cpu()
    ln = _ln32(hidden, mean, rstd, T)
    e_mean = h.mean(-1, keepdim=True)
    rs = ((h - e_mean).pow(2).mean(-1, keepdim=True) + EPS).rsqrt()
    xh = (h - e_mean) * rs
    s1 = _rd(1 + mods[:, 4 * D:5 * D].double()[:, None], T)
    dq = d_q.double()
    d_ln = _rd(dq * s1, T)
    c1, c2 = (xh * d_ln).mean(-1, keepdim=True), d_ln.mean(-1, keepdim=True)
    gr = (d_ln - (xh * c1 + c2)) * rs
    M_g = (d_ln.abs() + xh.abs() * (xh * d_ln).abs().mean(-1, keepdim=True) + d_ln.abs().mean(-1, keepdim=True)) * rs
    dh0 = d_hid.double() if with_dh else torch.zeros_like(gr)
    # dh = round(d_hidden + round(g)): the inner rounding in the reference too (the element counts as a mismatch only where
    # the fp32 error of g cannot move that rounding: conditioned)
    e_dx = dh0 + _rd(gr, T)
    check_elem(f"{tag} d_x", xd.grad, e_dx, dh0.abs() + M_g, max_ulp=2, extra=ulp(gr, T) if T in LOWP else None, conditioned=True)
    dh = xd.grad.detach().double().cpu()                    # d_mix / dgate from the kernel's own dh (its d_x), as ref_gated
    gate = mods[:, 2 * D:3 * D].double()[:, None]
    e_mix = torch.empty_like(dh)
    e_mix[:, src] = gate * dh
    check_elem(f"{tag} d_mix", mixd.grad, e_mix, e_mix.abs())
    dm = md.grad.double().cpu()
    check_colsum(f"{tag} dgate", md.grad[:, 2 * D:3 * D], (dh * mix[:, src].double()).sum(1), (dh * mix[:, src].double()).abs().sum(1))
    check_colsum(f"{tag} dshift", md.grad[:, 3 * D:4 * D], dq.sum(1), dq.abs().sum(1))
    check_colsum(f"{tag} dscale", md.grad[:, 4 * D:5 * D], (dq * ln).sum(1), (dq * ln).abs().sum(1))
    for j in (0, 1, 5):
        assert not dm[:, j * D:(j + 1) * D].any(), j
    return xd.grad, mixd.grad, md.grad


BWD_WIDTHS = (64, 368, 640, 768, 1024)              # MAXQ 4, 4, 5, 6, 8
# (B, L, row table, d_hidden): (3, 37) warp ranges straddle a batch boundary, (9, 5) one warp spans several batch elements,
# (4, 256) a longer sequence per element
BWD_CONFIGS = ((3, 37, "zigzag", True), (9, 5, "none", True), (4, 256, "temporal", False), (2, 64, "none", True))


@gpu
@pytest.mark.parametrize("D", BWD_WIDTHS)
@pytest.mark.parametrize("T", DTYPES, ids=[DTYPE_NAME[t] for t in DTYPES])
def test_backward_vs_fp64(T, D):
    for k, (B, L, kind, with_dh) in enumerate(BWD_CONFIGS):
        for det in (False, True):
            _bwd_case(T, D, B, L, kind, det, seed=31 * D + k, with_dh=with_dh)


@gpu
@pytest.mark.parametrize("T", DTYPES, ids=[DTYPE_NAME[t] for t in DTYPES])
def test_det_equals_atomic_and_repeats_bitwise(T):
    """The _det twin's gradients meet the same fp64 bounds as the atomic kernel's (checked inside _bwd_case; the column sums
    differ only in summation order) and repeat bit for bit; the row outputs (d_x, d_mix) are bitwise the same in both."""
    B, L, D = 16, 256, 768
    atomic = _bwd_case(T, D, B, L, "zigzag", False, seed=5)
    det = [_bwd_case(T, D, B, L, "zigzag", True, seed=5) for _ in range(2)]
    for a, b in zip(det[0], det[1]):
        assert torch.equal(a, b)
    assert torch.equal(atomic[0], det[0][0]) and torch.equal(atomic[1], det[0][1])


@gpu
@pytest.mark.parametrize("T", DTYPES, ids=[DTYPE_NAME[t] for t in DTYPES])
def test_batch_row_equals_row_alone(T):
    """Forward outputs and the row gradients of one batch element do not depend on the other elements."""
    from zigma_b200.engine import text_prologue
    B, L, D = 5, 64, 768
    x, mix, mods, table, _ = _inputs(B, L, D, T, 1, "zigzag", seed=3)
    md = mods.to(DEV)
    rowmap = table.to(torch.int32).to(DEV)
    full = text_prologue(x.to(DEV), mix.to(DEV), md[:, 2 * D:3 * D], md[:, 3 * D:4 * D], md[:, 4 * D:5 * D], rowmap, EPS)
    for r in (0, 3):
        one = text_prologue(x[r:r + 1].to(DEV), mix[r:r + 1].to(DEV), md[r:r + 1, 2 * D:3 * D], md[r:r + 1, 3 * D:4 * D],
                            md[r:r + 1, 4 * D:5 * D], rowmap, EPS)
        assert torch.equal(full[0][r:r + 1], one[0]) and torch.equal(full[1][r:r + 1], one[1]), (T, r)


@gpu
def test_matrix_reaches_every_instantiation():
    """The widths above launch every forward (T x Q 1..4) and backward (T x MAXQ 4/5/6/8 x DET) instantiation."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for T in DTYPES:
            for D in FWD_WIDTHS:
                _fwd_case(T, D, 2, 8, 1, "none", seed=D)
            for D in BWD_WIDTHS:
                for det in (False, True):
                    _bwd_case(T, D, 2, 8, "none", det, seed=D)
        torch.cuda.synchronize()
    names = {e.name for e in prof.events() if e.device_type.name == "CUDA" and "text_prologue" in e.name}
    fwd = {n for n in names if "text_prologue_fwd_kernel" in n}
    bwd = {n for n in names if "text_prologue_bwd_kernel" in n}
    assert len(fwd) == 12 and len(bwd) == 24, (sorted(fwd), sorted(bwd))


# ------------------------------------------------------------------------------------------------ model level
def _model(name, dtype=torch.float32, **over):
    from oracle import synth
    from zigma_b200 import ZigMa
    g, cfg, shapes = model_case(name)
    cfg = dict(cfg, **over)
    m = ZigMa(device=DEV, dtype=dtype, **cfg)
    m.load_state_dict(synth.synth_state_dict({k: tuple(v.shape) for k, v in m.state_dict().items()}, seed=0,
                                             **({} if dtype == torch.float32 else {"dtype": dtype})))
    return g, cfg, m


def _fused_vs_loop(m, cfg, x, tt, y, target, monkeypatch, autocast=False, spy=None):
    res = {}
    for mode in ("1", "0"):
        monkeypatch.setenv("ZIGMA_FUSED_TRAIN_TAIL", mode)
        assert m._fused_tail_ok(torch.empty(1, 1, cfg["embed_dim"], device=DEV)) == (mode == "1")
        for p_ in m.parameters():
            p_.grad = None
        if spy is not None:
            spy.clear()
        torch.manual_seed(1234)
        with torch.autocast("cuda", dtype=torch.bfloat16, enabled=autocast):
            out = m.forward_autograd(x, tt, y)
        rng = torch.cuda.get_rng_state()
        ((out.float() - target) ** 2).mean().backward()
        res[mode] = (out.detach().float(), {k: v.grad.clone().float() for k, v in m.named_parameters() if v.grad is not None}, rng,
                     None if spy is None else list(spy))
    return res


@gpu
@pytest.mark.parametrize("name", ["tiny_text", "tiny_video_text"])
def test_fused_training_loop_matches_per_op_loop_fp32(name, monkeypatch):
    """forward_autograd on the fused loop (text blocks included) vs ZIGMA_FUSED_TRAIN_TAIL=0: output and every parameter
    gradient at test_gpu_bwd.py's fp32 tolerances; the fused forward also against the reference golden."""
    from oracle import synth
    from oracle.gen_golden import model_io
    g, cfg, m = _model(name)
    m.eval()
    x, tt, y = model_io(cfg, g["out"].shape[0])
    target = synth.synth_latents(tuple(g["out"].shape), seed=77).to(DEV)
    res = _fused_vs_loop(m, cfg, x.to(DEV), tt.to(DEV), y.to(DEV), target, monkeypatch)
    check_close(res["1"][0], res["0"][0], f"{name} fused forward", atol=2e-5)
    check_close(res["1"][0], g["out"], f"{name} fused forward vs reference golden", atol=2e-5)
    assert set(res["1"][1]) == set(res["0"][1])
    assert any(".msa." in k for k in res["1"][1]) and any("adaLN" in k for k in res["1"][1])
    for k in res["0"][1]:
        check_close(res["1"][1][k], res["0"][1][k], f"{name} fused d{k}", atol=2e-5, max_strict_viol=2e-2)


@gpu
@pytest.mark.parametrize("name", ["tiny_text", "tiny_video_text"])
@pytest.mark.parametrize("mode", ["autocast", "bf16_params"])
def test_fused_training_loop_matches_per_op_loop_bf16(name, mode, monkeypatch):
    """The same comparison under bf16 autocast with fp32 parameters, and with bf16 parameters, at the whole-model bf16
    tolerance of test_gpu_model.py."""
    from oracle import synth
    from oracle.gen_golden import model_io
    g, cfg, m = _model(name, dtype=torch.bfloat16 if mode == "bf16_params" else torch.float32)
    m.eval()
    x, tt, y = model_io(cfg, g["out"].shape[0])
    cast = (lambda t: t.to(DEV).bfloat16()) if mode == "bf16_params" else (lambda t: t.to(DEV))
    target = synth.synth_latents(tuple(g["out"].shape), seed=77).to(DEV)
    res = _fused_vs_loop(m, cfg, cast(x), cast(tt), cast(y), target, monkeypatch, autocast=mode == "autocast")
    check_close(res["1"][0], res["0"][0], f"{name} {mode} fused forward", rtol=6e-2, atol=6e-2, scale_atol=True, max_strict_viol=1.0)
    assert set(res["1"][1]) == set(res["0"][1])
    for k in res["0"][1]:
        check_close(res["1"][1][k], res["0"][1][k], f"{name} {mode} fused d{k}", rtol=6e-2, atol=6e-2, scale_atol=True, max_strict_viol=1.0)


@gpu
@pytest.mark.parametrize("name", ["tiny_text", "tiny_video_text"])
def test_train_mode_drop_path_matches_per_op_loop(name, monkeypatch):
    """Train mode at drop-path rate 0.6: the same DropPath draws and CUDA generator state on both paths, output and every
    parameter gradient at the fp32 tolerances (the pattern of test_gpu_drop_path.py)."""
    from oracle.gen_golden import model_io
    from zigma_b200.model_zigma import DropPath
    g, cfg, m = _model(name, depth=4, drop_path_rate=0.6)
    m.train()
    x, tt, y = model_io(cfg, 8)
    x, tt, y = x.to(DEV), tt.to(DEV), y.to(DEV)
    with torch.no_grad():
        shape = m.forward_autograd(x, tt, y).shape
    target = torch.randn(shape, generator=torch.Generator().manual_seed(77)).to(DEV)
    drawn = []
    orig = DropPath.draw

    def spy(self, x_):
        mask = orig(self, x_)
        drawn.append(mask.flatten().cpu())
        return mask
    monkeypatch.setattr(DropPath, "draw", spy)
    res = _fused_vs_loop(m, cfg, x, tt, y, target, monkeypatch, spy=drawn)
    assert torch.equal(res["1"][2], res["0"][2]), "the two paths left the CUDA generator in different states"
    assert len(res["1"][3]) == len(res["0"][3]) and all(torch.equal(a, b) for a, b in zip(res["1"][3], res["0"][3]))
    assert any((mk == 0).any() and (mk != 0).any() for mk in res["1"][3][:-1]), "no block dropped one sample and kept another"
    check_close(res["1"][0], res["0"][0], f"{name} train-mode fused forward", atol=2e-5)
    for k in res["0"][1]:
        check_close(res["1"][1][k], res["0"][1][k], f"{name} train-mode fused d{k}", atol=2e-5, max_strict_viol=2e-2)


def _kernel_counts(fn):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    counts = {}
    for e in prof.events():
        if e.device_type.name == "CUDA":
            counts[e.name] = counts.get(e.name, 0) + 1
    return counts


# ATen kernels of the eager text branch the prologue replaces: the un-permuting gather, the gated add, norm_msa, modulate
_EAGER = ("layer_norm", "index_select", "indexselect", "index_kernel", "mulfunctor", "addfunctor", "cudafunctor_add")


def _per_block(counts_a, counts_b, depth_a, depth_b):
    """Launches per block of every kernel name: the count difference of two depths over the depth difference."""
    return {k: (counts_b.get(k, 0) - counts_a.get(k, 0)) / (depth_b - depth_a) for k in set(counts_a) | set(counts_b)}


@gpu
def test_profiler_prologue_kernels_per_block(monkeypatch):
    """An engine forward and a training step of a has_text model launch the prologue kernels once per block, _fused_tail_ok
    holds, and per block no ATen layer_norm or index_select kernel is left, nor, in the engine forward, any ATen mul / add
    (launch counts of depth 3 and depth 5 differ by none of them)."""
    from zigma_b200 import ZigMa
    g = torch.Generator(device=DEV).manual_seed(2)
    x = torch.randn(2, 4, 8, 8, device=DEV, generator=g).bfloat16()
    t = torch.rand(2, device=DEV, generator=g).bfloat16()
    y = torch.randn(2, 77, 24, device=DEV, generator=g).bfloat16()
    monkeypatch.setenv("ZIGMA_CUDA_GRAPH", "0")
    eng, train = {}, {}
    for depth in (3, 5):
        torch.manual_seed(0)
        # (no stochastic depth: its per-block mask arithmetic is not the text branch's)
        m = ZigMa(in_channels=4, embed_dim=128, depth=depth, img_dim=8, patch_size=1, scan_type="zigzagN8", num_classes=-1, has_text=True,
                  d_context=24, use_pe=2, drop_path_rate=0.0, device=DEV, dtype=torch.bfloat16).eval()
        with torch.no_grad():
            for p in m.parameters():
                if p.abs().sum() == 0:           # adaLN-zero init would silence both branches
                    p.normal_(0, 0.05)
            m(x, t, y)
            eng[depth] = _kernel_counts(lambda: m(x, t, y))
        m.train()
        assert m._fused_tail_ok(torch.empty(1, 1, 128, device=DEV, dtype=torch.bfloat16))
        m.forward_autograd(x, t, y).float().square().mean().backward()
        train[depth] = _kernel_counts(lambda: m.forward_autograd(x, t, y).float().square().mean().backward())
        for c in (eng[depth], train[depth]):
            assert sum(n for k, n in c.items() if "text_prologue_fwd_kernel" in k) == depth, c
        assert sum(n for k, n in train[depth].items() if "text_prologue_bwd_kernel" in k) == depth, train[depth]
        assert not [k for k in eng[depth] if "text_prologue_bwd" in k]
    # training: autograd's own gradient accumulation adds (the text tokens and c feed every block) are per-block ATen adds
    # that no fused kernel removes, so there only the normalisation and gather kernels of the per-op text branch are counted
    for what, c, names in (("engine forward", eng, _EAGER), ("training step", train, _EAGER[:4])):
        per = _per_block(c[3], c[5], 3, 5)
        left = {k: n for k, n in per.items() if n and any(s in k.lower() for s in names)}
        assert not left, (what, left)


@gpu
def test_engine_matches_forward_autograd():
    """The engine's text branch against forward_autograd (the fused training loop) in bf16, on every row-table case the
    engine has: zigzag image layers, and the spatial (B fold rows) and copy-free temporal (composite table) layers of a
    video model."""
    from oracle.gen_golden import model_io
    for name in ("tiny_text", "tiny_video_text"):
        g, cfg, m = _model(name, dtype=torch.bfloat16)
        m.eval()
        x, tt, y = model_io(cfg, 2)
        with torch.no_grad():
            eng_out = m(x.to(DEV).bfloat16(), tt.to(DEV).bfloat16(), y.to(DEV).bfloat16()).float()
            loop = m.forward_autograd(x.to(DEV).bfloat16(), tt.to(DEV).bfloat16(), y.to(DEV).bfloat16()).float()
        assert m._engine is not None
        check_close(eng_out, loop, f"{name} bf16 engine vs forward_autograd", rtol=6e-2, atol=6e-2, scale_atol=True, max_strict_viol=1.0)
