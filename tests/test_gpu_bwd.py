"""GPU (H100): backward kernels (selective_scan_cuda.bwd / causal_conv1d_bwd / layer-norm bwd
replacements) against the reference's autograd gradients (golden) and the differentiable oracle."""
import numpy as np
import pytest
import torch

from oracle import synth, zigma_oracle as zo
from util import check_close, gold, model_case, t

pytestmark = pytest.mark.gpu
DEV = "cuda"


@pytest.mark.parametrize("name", ["t128_g1", "t131_g2", "e64_n16", "plain", "noz", "l1", "l16_many", "n4", "e128_g2_n16", "e96_l45_n16"])
def test_selective_scan_bwd_golden(name):
    """Gradients of selective_scan_fn vs autograd through the reference's selective_scan_ref
    (test_selective_scan.py:121-149 protocol; tolerances: the north-star rtol 1e-3 with a range-scaled
    absolute floor, see util.check_close)."""
    from zigma_b200 import selective_scan_fn
    g = gold("scan_" + name)
    Bt, E, L, N, G, hasD, hasz, hasb, sp = [int(v) for v in g["flags"]]
    req = {k: t(g[k], DEV).requires_grad_() for k in ("u", "delta", "A", "B", "C", "D", "z", "delta_bias")}
    Bm = req["B"] if G > 1 else req["B"][:, 0]
    Cm = req["C"] if G > 1 else req["C"][:, 0]
    out = selective_scan_fn(req["u"], req["delta"], req["A"], Bm, Cm, req["D"] if hasD else None, z=req["z"] if hasz else None,
                            delta_bias=req["delta_bias"] if hasb else None, delta_softplus=bool(sp))
    check_close(out, g["out"], f"{name} out (grad mode)")
    out.backward(t(g["g"], DEV))
    names = ["u", "delta", "A", "B", "C"] + (["D"] if hasD else []) + (["z"] if hasz else []) + (["delta_bias"] if hasb else [])
    for k in names:
        check_close(req[k].grad, g["d" + k], f"{name} d{k}", atol=1e-4, max_strict_viol=1e-2)


@pytest.mark.parametrize("name", ["t128_g1", "t131_g2", "noz", "e128_g2_n16", "e96_l45_n16"])
def test_selective_scan_bwd_token_major(name):
    """Same golden gradients with every activation handed over TOKEN-MAJOR ((b, l, d) storage viewed as
    (b, d, l), the engine's layout): the dstate == 16 backward takes the strides as they come."""
    from zigma_b200 import selective_scan_fn
    g = gold("scan_" + name)
    Bt, E, L, N, G, hasD, hasz, hasb, sp = [int(v) for v in g["flags"]]
    tm = lambda a: t(a, DEV).transpose(-1, -2).contiguous().transpose(-1, -2).requires_grad_()
    req = {k: (tm(g[k]) if k in ("u", "delta", "z", "B", "C") else t(g[k], DEV).requires_grad_())
           for k in ("u", "delta", "A", "B", "C", "D", "z", "delta_bias")}
    assert req["u"].stride(1) == 1 and req["B"].stride(2) == 1
    Bm = req["B"] if G > 1 else req["B"][:, 0]
    Cm = req["C"] if G > 1 else req["C"][:, 0]
    out = selective_scan_fn(req["u"], req["delta"], req["A"], Bm, Cm, req["D"] if hasD else None, z=req["z"] if hasz else None,
                            delta_bias=req["delta_bias"] if hasb else None, delta_softplus=bool(sp))
    check_close(out, g["out"], f"{name} out (token-major, grad mode)")
    out.backward(t(g["g"], DEV).transpose(1, 2).contiguous().transpose(1, 2))
    names = ["u", "delta", "A", "B", "C"] + (["D"] if hasD else []) + (["z"] if hasz else []) + (["delta_bias"] if hasb else [])
    for k in names:
        check_close(req[k].grad, g["d" + k], f"{name} token-major d{k}", atol=1e-4, max_strict_viol=1e-2)


def test_selective_scan_bwd_bf16():
    from zigma_b200 import selective_scan_fn
    Bt, E, L, N = 2, 96, 150, 16
    inp = synth.synth_scan_inputs(Bt, E, L, N, 1, seed=21)
    lo = {k: (v.bfloat16() if k in ("u", "delta", "z", "B", "C") else v.clone()) for k, v in inp.items()}
    gout = torch.randn(Bt, E, L).bfloat16()
    ref_in = {k: v.float().clone().requires_grad_() for k, v in lo.items()}
    out_ref = zo.selective_scan(ref_in["u"], ref_in["delta"], ref_in["A"], ref_in["B"], ref_in["C"], ref_in["D"], ref_in["z"], ref_in["delta_bias"], True)
    out_ref.backward(gout.float())
    d = {k: v.detach().to(DEV).requires_grad_() for k, v in lo.items()}
    out = selective_scan_fn(d["u"], d["delta"], d["A"], d["B"], d["C"], d["D"], z=d["z"], delta_bias=d["delta_bias"], delta_softplus=True)
    out.backward(gout.to(DEV))
    for k in ("u", "delta", "z"):
        check_close(d[k].grad, ref_in[k].grad, f"bf16 d{k}", rtol=2e-2, atol=2e-2, scale_atol=True, max_strict_viol=1.0)
    for k in ("A", "D", "delta_bias"):
        check_close(d[k].grad, ref_in[k].grad, f"bf16 d{k} (fp32 accumulators)", rtol=1e-2, atol=1e-3, max_strict_viol=1.0)
    for k in ("B", "C"):
        check_close(d[k].grad, ref_in[k].grad, f"bf16 d{k}", rtol=2e-2, atol=2e-2, max_strict_viol=1.0)


def test_mamba_inner_fn_backward_vs_oracle_autograd():
    from zigma_b200 import mamba_inner_fn
    g = gold("mamba_inner")
    names = ["xz", "conv_w", "conv_b", "x_proj_w", "dt_proj_w", "out_proj_w", "out_proj_b", "A", "D", "delta_bias"]
    ref = {k: t(g[k]).requires_grad_() for k in names}
    o_ref = zo.mamba_inner(*[ref[k] for k in names])
    gout = torch.from_numpy(np.random.RandomState(3).randn(*o_ref.shape).astype(np.float32))
    o_ref.backward(gout)
    a = {k: t(g[k], DEV).requires_grad_() for k in names}
    out = mamba_inner_fn(a["xz"], a["conv_w"], a["conv_b"], a["x_proj_w"], a["dt_proj_w"], a["out_proj_w"], a["out_proj_b"],
                         a["A"], None, None, a["D"], a["delta_bias"], delta_softplus=True)
    check_close(out, o_ref, "mamba_inner_fn fwd (grad mode)")
    out.backward(gout.to(DEV))
    for k in names:
        check_close(a[k].grad, ref[k].grad, f"mamba_inner_fn d{k}", atol=1e-4, max_strict_viol=2e-2)


@pytest.mark.parametrize("name", ["tiny_zigzag8", "tiny_sweep2", "tiny_video_sst"])
def test_zigma_training_step_gradients(name):
    """One flow-matching training step (MSE to a target velocity) through ZigMa.forward_autograd:
    parameter gradients vs autograd through the CPU oracle with the same weights."""
    from zigma_b200 import ZigMa
    from oracle.gen_golden import model_io
    g, cfg, shapes = model_case(name)
    sd = synth.synth_state_dict(shapes, seed=0)
    m = ZigMa(device=DEV, **cfg).eval()      # eval: drop_path off (stochastic), gradients still flow
    m.load_state_dict(sd)
    x, tt, y = model_io(cfg, g["out"].shape[0])
    target = synth.synth_latents(tuple(g["out"].shape), seed=77)
    out = m.forward_autograd(x.to(DEV), tt.to(DEV), None if y is None else y.to(DEV))
    check_close(out, g["out"], f"{name} forward_autograd", atol=2e-5)
    loss = ((out - target.to(DEV)) ** 2).mean()
    loss.backward()
    sdr = {k: v.clone().requires_grad_() for k, v in sd.items()}
    out_ref = zo.zigma_forward(sdr, dict(cfg, norm_epsilon=1e-5), x, tt, y)
    ((out_ref - target) ** 2).mean().backward()
    params = dict(m.named_parameters())
    checked = 0
    for k, v in sdr.items():
        if v.grad is None or k not in params:
            continue
        check_close(params[k].grad, v.grad, f"{name} grad {k}", rtol=2e-3, atol=2e-5, max_strict_viol=5e-2)
        checked += 1
    assert checked >= 20


@pytest.mark.parametrize("scan_type,dtype", [("zigzagN8", torch.float32), ("v1", torch.float32), ("zigzagN8", torch.bfloat16)])
def test_mamba_token_major_path_matches_channel_first(scan_type, dtype, monkeypatch):
    """Mamba.forward through the token-major training core (permutation fused into conv / scan forward AND
    backward kernels) vs the reference-layout branch (gather -> mamba_inner_fn -> gather): outputs, input
    gradient and every parameter gradient."""
    from zigma_b200.mamba_simple import Mamba
    from zigma_b200 import zigzag_path, reverse_permut_np
    side, dm, bs = 12, 48, 3
    L = side * side
    paths = zigzag_path(side)
    kw = {}
    if scan_type != "v1":
        kw = dict(zigzag_paths=[torch.from_numpy(np.ascontiguousarray(p)).to(DEV) for p in paths],
                  zigzag_paths_reverse=[torch.from_numpy(np.ascontiguousarray(reverse_permut_np(p))).to(DEV) for p in paths])
    torch.manual_seed(0)
    m = Mamba(dm, d_state=16, layer_idx=3, device=DEV, dtype=dtype, scan_type=scan_type, **kw)
    x = torch.randn(bs, L, dm, device=DEV, dtype=dtype)
    gout = torch.randn(bs, L, dm, device=DEV, dtype=dtype)
    res = {}
    for mode in ("1", "0"):
        monkeypatch.setenv("ZIGMA_TOKEN_MAJOR_TRAIN", mode)
        for p_ in m.parameters():
            p_.grad = None
        xi = x.clone().requires_grad_()
        out = m(xi)
        out.backward(gout)
        res[mode] = (out.detach(), xi.grad, {k: v.grad.clone() for k, v in m.named_parameters() if v.grad is not None})
    assert m._tok_eligible(x) is False            # env still "0" here; and the two runs really took different branches
    lo = dtype == torch.bfloat16
    tol = dict(rtol=3e-2, atol=3e-2, scale_atol=True, max_strict_viol=1.0) if lo else dict(atol=2e-5, max_strict_viol=1e-2)
    check_close(res["1"][0], res["0"][0], f"{scan_type} token-major out", **tol)
    check_close(res["1"][1], res["0"][1], f"{scan_type} token-major dx", **tol)
    assert set(res["1"][2]) == set(res["0"][2]) and len(res["1"][2]) >= 9
    for k in res["0"][2]:
        check_close(res["1"][2][k], res["0"][2][k], f"{scan_type} token-major d{k}", **tol)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_scan_bwd_staged_kernel_groups_rowmap_vs_oracle_autograd(dtype):
    """The cp.async-staged dstate-16 backward (whole 64-channel tiles, L % 8 == 0): two groups, both layouts, and the
    fused z permutation (z_rowmap) -- against autograd through the CPU oracle on gathered inputs."""
    from zigma_b200.selective_scan_interface import _scan_fwd, _scan_bwd
    Bt, E, L, N, G = 2, 128, 72, 16, 2
    inp = synth.synth_scan_inputs(Bt, E, L, N, G, seed=31)
    lo = {k: (v.to(dtype) if k in ("u", "delta", "z", "B", "C") else v.clone()) for k, v in inp.items()}
    perm = torch.randperm(L, generator=torch.Generator().manual_seed(5))
    gout = torch.randn(Bt, E, L, generator=torch.Generator().manual_seed(6)).to(dtype)
    ref = {k: v.float().clone().requires_grad_() for k, v in lo.items()}
    out_ref = zo.selective_scan(ref["u"], ref["delta"], ref["A"], ref["B"], ref["C"], ref["D"], ref["z"][:, :, perm], ref["delta_bias"], True)
    out_ref.backward(gout.float())
    tm = lambda a: a.transpose(-1, -2).contiguous().transpose(-1, -2)
    d = {k: v.to(DEV) for k, v in lo.items()}
    tol = dict(rtol=3e-2, atol=3e-2, max_strict_viol=1.0) if dtype == torch.bfloat16 else dict(atol=1e-4, max_strict_viol=1e-2)
    for layout in ("tok", "seq"):
        if layout == "tok":
            u, dl, z, B, C, go = tm(d["u"]), tm(d["delta"]), tm(d["z"]), tm(d["B"]), tm(d["C"]), tm(gout.to(DEV))
            rowmap = perm.to(DEV).to(torch.int32)
        else:   # channel-first has no rowmap: hand over the gathered z and scatter dz afterwards
            u, dl, z, B, C, go = d["u"], d["delta"], d["z"][:, :, perm.to(DEV)].contiguous(), d["B"], d["C"], gout.to(DEV)
            rowmap = None
        out, _, ckpt, saved = _scan_fwd(u, dl, d["A"], B, C, d["D"], z, d["delta_bias"], True, z_rowmap=rowmap, want_last_state=False, want_ckpt=True)
        check_close(out, out_ref, f"staged {layout} fwd(+ckpt)", **tol)
        du, ddl, dA, dB, dC, dD, dbias, dz = _scan_bwd(saved, ckpt, go, True, z_rowmap=rowmap)
        if layout == "seq":
            full = torch.empty_like(dz); full[:, :, perm.to(DEV)] = dz; dz = full
        for name, got, want in (("du", du, ref["u"].grad), ("ddelta", ddl, ref["delta"].grad), ("dz", dz, ref["z"].grad), ("dA", dA, ref["A"].grad),
                                ("dB", dB, ref["B"].grad), ("dC", dC, ref["C"].grad), ("dD", dD, ref["D"].grad), ("dbias", dbias, ref["delta_bias"].grad)):
            check_close(got, want, f"staged {layout} {name}", **tol)


@pytest.mark.parametrize("const_b,const_c", [(True, False), (False, True), (True, True)])
@pytest.mark.parametrize("N", [4, 16])
def test_selective_scan_bwd_constant_bc_vs_oracle_autograd(const_b, const_c, N):
    """Constant (dim, dstate) fp32 B and / or C (the non input-dependent forms selective_scan.cpp:238-278 accepts; their
    gradients are per-channel sums over batch and sequence, selective_scan_bwd_kernel.cuh:297-316) through the public
    selective_scan_fn, against autograd through the CPU oracle."""
    from zigma_b200 import selective_scan_fn
    Bt, E, L = 2, 96, 45
    inp = synth.synth_scan_inputs(Bt, E, L, N, 1, seed=41)
    g = torch.Generator().manual_seed(7)
    if const_b:
        inp["B"] = torch.randn(E, N, generator=g) * 0.5
    if const_c:
        inp["C"] = torch.randn(E, N, generator=g) * 0.5
    gout = torch.randn(Bt, E, L, generator=g)
    ref = {k: v.float().clone().requires_grad_() for k, v in inp.items()}
    out_ref = zo.selective_scan(ref["u"], ref["delta"], ref["A"], ref["B"], ref["C"], ref["D"], ref["z"], ref["delta_bias"], True)
    out_ref.backward(gout)
    d = {k: v.to(DEV).requires_grad_() for k, v in inp.items()}
    out = selective_scan_fn(d["u"], d["delta"], d["A"], d["B"], d["C"], d["D"], z=d["z"], delta_bias=d["delta_bias"], delta_softplus=True)
    check_close(out, out_ref, f"constant B={const_b} C={const_c} N={N} fwd", atol=1e-4, max_strict_viol=1e-2)
    out.backward(gout.to(DEV))
    for k in ("u", "delta", "z", "A", "B", "C", "D", "delta_bias"):
        assert d[k].grad.shape == ref[k].grad.shape and d[k].grad.dtype == d[k].dtype
        check_close(d[k].grad, ref[k].grad, f"constant B={const_b} C={const_c} N={N} d{k}", atol=1e-4, max_strict_viol=1e-2)


@pytest.mark.parametrize("N", [24, 32, 64])
def test_selective_scan_bwd_wide_state_vs_oracle_autograd(N):
    """dstate up to 64 in the backward (what the forward accepts; the reference takes up to 256, selective_scan.cpp:262), generic
    kernel: against autograd through the CPU oracle."""
    from zigma_b200 import selective_scan_fn
    Bt, E, L = 2, 64, 40
    inp = synth.synth_scan_inputs(Bt, E, L, N, 1, seed=43)
    gout = torch.randn(Bt, E, L, generator=torch.Generator().manual_seed(8))
    ref = {k: v.float().clone().requires_grad_() for k, v in inp.items()}
    out_ref = zo.selective_scan(ref["u"], ref["delta"], ref["A"], ref["B"], ref["C"], ref["D"], ref["z"], ref["delta_bias"], True)
    out_ref.backward(gout)
    d = {k: v.to(DEV).requires_grad_() for k, v in inp.items()}
    out = selective_scan_fn(d["u"], d["delta"], d["A"], d["B"], d["C"], d["D"], z=d["z"], delta_bias=d["delta_bias"], delta_softplus=True)
    check_close(out, out_ref, f"dstate {N} fwd", atol=1e-4, max_strict_viol=1e-2)
    out.backward(gout.to(DEV))
    for k in ("u", "delta", "z", "A", "B", "C", "D", "delta_bias"):
        check_close(d[k].grad, ref[k].grad, f"dstate {N} d{k}", atol=1e-4, max_strict_viol=1e-2)


def test_scan_bwd_full_size_properties():
    """BASELINE config-2 layer shape (bs 16 x 1280 x 1024, bf16, token-major): (a) every gradient is linear in dout --
    bwd(2 dout) == 2 bwd(dout) exactly for the per-element outputs (power-of-two scaling commutes with every rounding),
    (b) the first half of the batch gives bit-identical du / ddelta / dz when the second half of every input changes."""
    from zigma_b200.selective_scan_interface import _scan_fwd, _scan_bwd
    bs, E, L, N = 16, 1280, 1024, 16
    g = torch.Generator(device=DEV).manual_seed(0)
    dt = torch.bfloat16
    mk = lambda *s: torch.randn(*s, device=DEV, generator=g).to(dt)
    u, z, dout = mk(bs, L, E).transpose(1, 2), mk(bs, L, E).transpose(1, 2), mk(bs, L, E).transpose(1, 2)
    delta = (0.5 * torch.rand(bs, L, E, device=DEV, generator=g)).to(dt).transpose(1, 2)
    B, C = mk(bs, 1, L, N).transpose(2, 3), mk(bs, 1, L, N).transpose(2, 3)
    A = -0.5 * torch.rand(E, N, device=DEV, generator=g); D = torch.randn(E, device=DEV, generator=g); bias = 0.5 * torch.rand(E, device=DEV, generator=g)
    _, _, ckpt, saved = _scan_fwd(u, delta, A, B, C, D, z, bias, True, want_last_state=False, want_ckpt=True)
    r1 = _scan_bwd(saved, ckpt, dout, True)
    r2 = _scan_bwd(saved, ckpt, dout * 2, True)
    for i, name in ((0, "du"), (1, "ddelta"), (7, "dz")):
        assert torch.equal(r2[i].float(), 2 * r1[i].float()), name
    check_close(r2[3], 2 * r1[3], "dB linear", rtol=1e-4, atol=1e-3, max_strict_viol=1.0)      # (atomics: order-dependent last bits)
    u2, z2, dl2, do2 = u.clone(), z.clone(), delta.clone(), dout.clone()
    for t_ in (u2, z2, dl2, do2):
        t_[bs // 2:] = t_[bs // 2:].flip(0)
    B2, C2 = B.clone(), C.clone(); B2[bs // 2:] = B2[bs // 2:].flip(0); C2[bs // 2:] = C2[bs // 2:].flip(0)
    _, _, ck2, sv2 = _scan_fwd(u2, dl2, A, B2, C2, D, z2, bias, True, want_last_state=False, want_ckpt=True)
    r3 = _scan_bwd(sv2, ck2, do2, True)
    for i, name in ((0, "du"), (1, "ddelta"), (7, "dz")):
        assert torch.equal(r3[i][:bs // 2], r1[i][:bs // 2]), name + " batch slice"
        assert torch.equal(r3[i][bs // 2:], r1[i][bs // 2:].flip(0)), name + " flipped half"


@pytest.mark.parametrize("name", ["tiny_zigzag8", "tiny_sweep2", "tiny_video_sst"])
def test_fused_training_tail_matches_unfused_block_loop(name, monkeypatch):
    """ZigMa.forward_autograd with the fused block tails (ZIGMA_FUSED_TRAIN_TAIL=1, default) vs the per-op block loop:
    output and every parameter gradient (fp32)."""
    from zigma_b200 import ZigMa
    from oracle.gen_golden import model_io
    g, cfg, shapes = model_case(name)
    sd = synth.synth_state_dict(shapes, seed=0)
    m = ZigMa(device=DEV, **cfg).eval()
    m.load_state_dict(sd)
    x, tt, y = model_io(cfg, g["out"].shape[0])
    target = synth.synth_latents(tuple(g["out"].shape), seed=77).to(DEV)
    res = {}
    for mode in ("1", "0"):
        monkeypatch.setenv("ZIGMA_FUSED_TRAIN_TAIL", mode)
        for p_ in m.parameters():
            p_.grad = None
        out = m.forward_autograd(x.to(DEV), tt.to(DEV), None if y is None else y.to(DEV))
        ((out - target) ** 2).mean().backward()
        res[mode] = (out.detach(), {k: v.grad.clone() for k, v in m.named_parameters() if v.grad is not None})
    check_close(res["1"][0], res["0"][0], f"{name} fused-tail forward", atol=2e-5)
    check_close(res["1"][0], g["out"], f"{name} fused-tail forward vs reference golden", atol=2e-5)
    assert set(res["1"][1]) == set(res["0"][1])
    for k in res["0"][1]:
        check_close(res["1"][1][k], res["0"][1][k], f"{name} fused-tail d{k}", atol=2e-5, max_strict_viol=2e-2)
