"""GPU (H100): ZigMa.forward / mamba_inner_fn end to end against the golden vectors produced by the
unmodified reference, through both execution paths (engine fast path and autograd path)."""
import numpy as np
import pytest
import torch

from oracle import synth, zigma_oracle as zo
from oracle.gen_golden import model_io
from util import check_close, gold, model_case, t

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _build(cfg, shapes, dtype=torch.float32):
    from zigma_b200 import ZigMa
    m = ZigMa(device=DEV, dtype=dtype, **cfg).eval()
    sd = synth.synth_state_dict(shapes, seed=0, dtype=dtype)
    m.load_state_dict(sd, strict=True)
    return m, sd


def test_mamba_inner_fn_golden():
    from zigma_b200 import mamba_inner_fn
    g = gold("mamba_inner")
    a = {k: t(g[k], DEV) for k in g.files}
    out = mamba_inner_fn(a["xz"], a["conv_w"], a["conv_b"], a["x_proj_w"], a["dt_proj_w"], a["out_proj_w"], a["out_proj_b"],
                         a["A"], None, None, a["D"], a["delta_bias"], delta_softplus=True)
    check_close(out, g["out"], "mamba_inner_fn")
    # bimamba_inner_fn against the reference's bimamba_inner_ref (selective_scan_interface.py:673-711), forward and gradients
    from zigma_b200 import bimamba_inner_fn
    req = {k: a[k].clone().requires_grad_() for k in ("xz", "conv_w", "x_proj_w", "dt_proj_w", "out_proj_w", "A", "A_b", "D")}
    ob = bimamba_inner_fn(req["xz"], req["conv_w"], a["conv_b"], req["x_proj_w"], req["dt_proj_w"], req["out_proj_w"], a["out_proj_b"],
                          req["A"], req["A_b"], None, None, req["D"], a["delta_bias"], delta_softplus=True)
    check_close(ob, g["out_bi"], "bimamba_inner_fn vs bimamba_inner_ref")
    ob.square().sum().backward()
    assert all(v.grad is not None and torch.isfinite(v.grad).all() and v.grad.abs().sum() > 0 for v in req.values())


@pytest.mark.parametrize("name", ["tiny_zigzag8", "tiny_sweep2", "tiny_hilbert2", "tiny_patch2_cls", "tiny_video_sst", "tiny_text", "tiny_video_text"])
@pytest.mark.parametrize("path", ["engine", "engine_nograph", "autograd"])
def test_zigma_forward_golden_fp32(name, path, monkeypatch):
    g, cfg, shapes = model_case(name)
    m, _ = _build(cfg, shapes)
    x, tt, y = model_io(cfg, g["out"].shape[0])
    x, tt = x.to(DEV), tt.to(DEV)
    y = None if y is None else y.to(DEV)
    if path == "autograd":
        out = m.forward_autograd(x, tt, y)
    else:
        if path == "engine_nograph":
            monkeypatch.setenv("ZIGMA_CUDA_GRAPH", "0")
        with torch.no_grad():
            out = m(x, tt, y)
            if path == "engine":     # second call replays the captured graph
                out2 = m(x, tt, y)
                assert torch.equal(out, out2)
    check_close(out, g["out"], f"ZigMa.forward {name} [{path}]", atol=2e-5)


def test_zigma_forward_full_model_fp32():
    """BASELINE config-2 architecture (D=640, depth=18, 32x32, zigzag8) at bs=1, fp32, vs the reference."""
    g, cfg, shapes = model_case("full_zigzag8_b1")
    m, _ = _build(cfg, shapes)
    x, tt, y = model_io(cfg, 1)
    with torch.no_grad():
        out = m(x.to(DEV), tt.to(DEV))
    check_close(out, g["out"], "ZigMa.forward full zigzag8_b1 fp32", atol=2e-5)


def test_zigma_forward_bf16():
    """bf16 state dict (every parameter bf16, SURVEY.md section 8d): tiny model vs the reference's bf16 CPU
    output, and the bf16 result must also sit close to the fp32 result of the same weights."""
    g, cfg, shapes = model_case("tiny_zigzag8_bf16")
    m, sd = _build(cfg, shapes, torch.bfloat16)
    x, tt, y = model_io(cfg, g["out"].shape[0])
    with torch.no_grad():
        out = m(x.to(DEV).bfloat16(), tt.to(DEV).bfloat16())
    assert out.dtype == torch.bfloat16
    check_close(out, g["out"], "ZigMa.forward tiny bf16 vs reference bf16", rtol=5e-2, atol=5e-2, scale_atol=False, max_strict_viol=1.0)
    g32 = gold("model_tiny_zigzag8")
    check_close(out, g32["out"], "ZigMa.forward tiny bf16 vs reference fp32", rtol=5e-2, atol=5e-2, scale_atol=False, max_strict_viol=1.0)


def test_engine_pos_embed_folded_into_first_tail_bit_identical(monkeypatch):
    """The engine adds pos_embed inside its first fused tail (zg_block_tail_fwd_pe); ZIGMA_FOLD_PE=0 runs the eager add of
    ZigMa.embed (model_zigma.py:941) instead.  Same rounding point -> the two evaluations agree bit for bit; the folded one
    launches one zigma_b200 kernel of the same count (the add was a torch kernel) and stays on the reference's bf16 output."""
    from zigma_b200 import ZigMa
    g, cfg, shapes = model_case("tiny_zigzag8_bf16")
    assert cfg.get("use_pe", 0) in (1, 2)
    x, tt, y = model_io(cfg, g["out"].shape[0])
    outs = []
    for fold in ("1", "0"):
        monkeypatch.setenv("ZIGMA_FOLD_PE", fold)
        m, _ = _build(cfg, shapes, torch.bfloat16)
        with torch.no_grad():
            outs.append(m(x.to(DEV).bfloat16(), tt.to(DEV).bfloat16()))
    assert torch.equal(outs[0], outs[1])
    check_close(outs[0], g["out"], "ZigMa.forward tiny bf16, pos_embed folded", rtol=5e-2, atol=5e-2, scale_atol=False, max_strict_viol=1.0)


def test_zigma_forward_sweep2_bf16_fused_flip_add():
    """scan_type v2 in bf16: the engine folds `y_fwd + y_bwd.flip(1)` into the second scan kernel (OUT_REVERSE | OUT_ACCUMULATE)
    when the layer fits the hot-path kernel (D = 128 here: dt_rank 8, 16-byte aligned B / C columns); result vs the fp32 oracle
    on the same (bf16-rounded) weights at the whole-model bf16 tolerance.  D = 32 (dt_rank 2) takes the eager flip + add."""
    from zigma_b200 import ZigMa
    for D in (128, 32):
        cfg = dict(in_channels=4, embed_dim=D, depth=2, img_dim=8, patch_size=1, scan_type="v2", use_pe=2)
        m = ZigMa(device=DEV, dtype=torch.bfloat16, **cfg).eval()
        sd = synth.synth_state_dict({k: tuple(v.shape) for k, v in m.state_dict().items()}, seed=0, dtype=torch.bfloat16)
        m.load_state_dict(sd)
        x, tt, y = model_io(cfg, 2)
        with torch.no_grad():
            out = m(x.to(DEV).bfloat16(), tt.to(DEV).bfloat16())
        want = zo.zigma_forward({k: v.float() for k, v in sd.items()}, dict(cfg, norm_epsilon=1e-5), x.bfloat16().float(), tt.bfloat16().float())
        check_close(out, want, f"ZigMa.forward tiny v2 bf16 D={D} vs fp32 oracle", rtol=5e-2, atol=5e-2, scale_atol=False, max_strict_viol=1.0)


def test_zigma_forward_batch_consistency_bf16_full():
    """Full-size bf16 model at bs=4: each sample equals the bs=1 run of that sample (samples are
    independent -> the multi-GPU batch sharding cannot change results), output finite."""
    g, cfg, shapes = model_case("full_zigzag8_b1")
    m, _ = _build(cfg, shapes, torch.bfloat16)
    x = synth.synth_latents((4, 4, 32, 32), seed=5).to(DEV).bfloat16()
    tt = torch.tensor([0.1, 0.4, 0.6, 0.9], device=DEV).bfloat16()
    with torch.no_grad():
        out = m(x, tt)
        one = m(x[2:3], tt[2:3])
    assert torch.isfinite(out.float()).all()
    check_close(out[2:3], one, "bs=4 vs bs=1 sample", rtol=2e-2, atol=2e-2, scale_atol=False, max_strict_viol=1.0)
    # and against the fp32 reference golden for sample seed 3 at bs = 1
    x1, t1, _ = model_io(cfg, 1)
    with torch.no_grad():
        o1 = m(x1.to(DEV).bfloat16(), t1.to(DEV).bfloat16())
    check_close(o1, g["out"], "full model bf16 vs reference fp32", rtol=6e-2, atol=6e-2, scale_atol=False, max_strict_viol=1.0)


def test_euler_sampling_loop_matches_oracle():
    from zigma_b200 import create_transport, Sampler
    g, cfg, shapes = model_case("tiny_zigzag8")
    m, sd = _build(cfg, shapes)
    x0 = synth.synth_latents((2, 4, 8, 8), seed=8)
    fn = Sampler(create_transport()).sample_ode(sampling_method="euler", num_steps=6)
    with torch.no_grad():
        got = fn(x0.to(DEV), m.forward)[-1]
    ocfg = dict(cfg, norm_epsilon=1e-5)
    want = zo.sample_ode_fixed(lambda x, t: zo.zigma_forward(sd, ocfg, x, t), x0, num_steps=6)
    check_close(got, want, "5-step Euler sampling", atol=5e-5)


def test_whole_loop_graph_euler_matches_sampler_and_oracle():
    """ZigMa.sample_euler (the whole fixed-grid Euler loop as ONE CUDA-graph replay, SURVEY 8f-2) == the step-by-step
    Sampler.sample_ode("euler") == the oracle's loop around the oracle's forward."""
    from zigma_b200 import create_transport, Sampler
    g, cfg, shapes = model_case("tiny_zigzag8")
    m, sd = _build(cfg, shapes)
    x0 = synth.synth_latents((2, 4, 8, 8), seed=8)
    with torch.no_grad():
        traj = Sampler(create_transport()).sample_ode(sampling_method="euler", num_steps=6)(x0.to(DEV), m.forward)
        got = m.sample_euler(x0.to(DEV), num_steps=6)
        got_traj = m.sample_euler(x0.to(DEV), num_steps=6, return_trajectory=True)
        again = m.sample_euler(x0.to(DEV) * 1.0, num_steps=6)          # second call: pure replay
    assert torch.equal(got, again) and torch.equal(got_traj[-1], got) and got_traj.shape == traj.shape
    check_close(got, traj[-1], "whole-loop graph vs step-by-step sampler", atol=5e-5)
    ocfg = dict(cfg, norm_epsilon=1e-5)
    want = zo.sample_ode_fixed(lambda x, t: zo.zigma_forward(sd, ocfg, x, t), x0, num_steps=6)
    check_close(got, want, "whole-loop graph Euler vs oracle", atol=5e-5)


# ---- the other BASELINE.json configs at their real widths (parity-test cases, not bench lines) ---------------
def _oracle_forward(cfg, sd, x, t, y=None):
    """CPU oracle with the plain-C scan (fp32): seconds at bs=1 even for L = 4096."""
    zo.USE_C_SCAN = True
    try:
        return zo.zigma_forward(sd, dict(cfg, norm_epsilon=1e-5), x, t, y)
    finally:
        zo.USE_C_SCAN = False


FULL_WIDTH_CASES = {
    # BASELINE configs[2]: sweep2_b1 (scan_type "v2": two directional scans per layer, separate parameters)
    "config3_sweep2_b1": (dict(in_channels=4, embed_dim=640, depth=18, img_dim=32, patch_size=1, scan_type="v2", use_pe=2), (1, 4, 32, 32)),
    # BASELINE configs[3]: FacesHQ-1024 shape -- D=768, 128x128 latent, patch 2 -> L = 4096, zigzag tables of side 64
    # (depth cut from 24 to 4 to bound the CPU oracle's time; widths, L and tables are the real ones)
    "config4_faceshq1024": (dict(in_channels=4, embed_dim=768, depth=4, img_dim=128, patch_size=2, scan_type="zigzagN8", use_pe=0), (1, 4, 128, 128)),
    # BASELINE configs[4]: UCF101 3d_zigzag8sst_b2 shape -- 16 frames x (32/2)^2 tokens, s/s/t factorised scans,
    # 101 classes (depth cut from 24 to 6 = two s,s,t rounds)
    "config5_ucf101_sst": (dict(in_channels=4, embed_dim=768, depth=6, img_dim=32, patch_size=2, scan_type="zzvideo_sst", use_pe=2,
                                video_frames=16, tpe=True, num_classes=101), (1, 16, 4, 32, 32)),
}


@pytest.mark.parametrize("name", list(FULL_WIDTH_CASES))
def test_other_baseline_configs_fp32_vs_oracle(name):
    from zigma_b200 import ZigMa
    cfg, xshape = FULL_WIDTH_CASES[name]
    m = ZigMa(device=DEV, **cfg).eval()
    shapes = {k: tuple(v.shape) for k, v in m.state_dict().items()}
    sd = synth.synth_state_dict(shapes, seed=0)
    m.load_state_dict(sd)
    x = synth.synth_latents(xshape, seed=11)
    tt = torch.tensor([0.37])
    y = torch.tensor([42]) if cfg.get("num_classes", -1) > 0 else None
    with torch.no_grad():
        got = m(x.to(DEV), tt.to(DEV), None if y is None else y.to(DEV))
    want = _oracle_forward(cfg, sd, x, tt, y)
    check_close(got, want, f"{name} fp32 engine vs CPU oracle", atol=2e-5)


@pytest.mark.parametrize("name", ["config4_faceshq1024", "config5_ucf101_sst"])
def test_other_baseline_configs_bf16_batch(name):
    """bf16 at a multi-sample batch: finite, each sample equal to its bs=1 run, close to the fp32 oracle."""
    from zigma_b200 import ZigMa
    cfg, xshape = FULL_WIDTH_CASES[name]
    m = ZigMa(device=DEV, dtype=torch.bfloat16, **cfg).eval()
    shapes = {k: tuple(v.shape) for k, v in m.state_dict().items()}
    sd = synth.synth_state_dict(shapes, seed=0)
    m.load_state_dict({k: v.bfloat16() for k, v in sd.items()})
    bs = 3
    x = synth.synth_latents((bs,) + xshape[1:], seed=12)
    tt = torch.tensor([0.2, 0.5, 0.8])
    y = torch.tensor([3, 50, 100]) if cfg.get("num_classes", -1) > 0 else None
    with torch.no_grad():
        out = m(x.to(DEV).bfloat16(), tt.to(DEV).bfloat16(), None if y is None else y.to(DEV))
        one = m(x[1:2].to(DEV).bfloat16(), tt[1:2].to(DEV).bfloat16(), None if y is None else y[1:2].to(DEV))
    assert torch.isfinite(out.float()).all()
    check_close(out[1:2], one, f"{name} bf16 bs=3 vs bs=1", rtol=2e-2, atol=2e-2, scale_atol=False, max_strict_viol=1.0)
    want = _oracle_forward(cfg, sd, x[1:2], tt[1:2], None if y is None else y[1:2])
    check_close(one, want, f"{name} bf16 vs fp32 oracle", rtol=8e-2, atol=8e-2, scale_atol=False, max_strict_viol=1.0)


FULL_DEPTH_CASES = {
    # BASELINE configs[3] / configs[4] exactly as bench.py measures them (reference yaml hyper-parameters, depth 24), at half the
    # per-GPU batch of the benchmark (bs 16 / 8): the whole-batch bf16 engine path, checked on sampled rows against the fp32 oracle
    "faceshq1024": (dict(in_channels=4, embed_dim=768, depth=24, img_dim=128, patch_size=2, scan_type="zigzagN8"), (4, 128, 128), 16),
    "ucf101_sst": (dict(in_channels=4, embed_dim=768, depth=24, img_dim=32, patch_size=2, scan_type="zzvideo_sst", use_pe=2, video_frames=16,
                        num_classes=101), (16, 4, 32, 32), 16),
}


@pytest.mark.parametrize("name", list(FULL_DEPTH_CASES))
def test_full_depth_configs_bf16_batch16(name):
    """Full depth (24 blocks), bf16, bs = 16 -- the batch path of BASELINE configs 3 / 4 (L = 4096; 16 frames x 256 tokens with
    s / s / t scans: 4096 sequences of length 16 in the temporal layers), through the engine AND through the whole-loop
    CUDA-graph sampler.  Too big for the CPU oracle as a batch, so: finite everywhere; a sample of the batch equals its own
    bs = 1 run bit for bit (samples are independent: what multi-GPU sharding relies on); that sample agrees with the fp32 CPU
    oracle (C scan) at the whole-model bf16 tolerance."""
    from zigma_b200 import ZigMa
    cfg, lat, bs = FULL_DEPTH_CASES[name]
    m = ZigMa(device=DEV, dtype=torch.bfloat16, **cfg).eval()
    shapes = {k: tuple(v.shape) for k, v in m.state_dict().items()}
    sd = synth.synth_state_dict(shapes, seed=0)
    m.load_state_dict({k: v.bfloat16() for k, v in sd.items()})
    x = synth.synth_latents((bs,) + lat, seed=21).bfloat16()
    tt = torch.linspace(0.05, 0.95, bs).bfloat16()
    y = (torch.arange(bs) * 7) % 101 if cfg.get("num_classes", -1) > 0 else None
    k = 11                                                   # the sampled row of the batch
    yd = None if y is None else y.to(DEV)
    with torch.no_grad():
        out = m(x.to(DEV), tt.to(DEV), yd)
        one = m(x[k:k + 1].to(DEV), tt[k:k + 1].to(DEV), None if y is None else yd[k:k + 1])
        step = m.sample_euler(x.to(DEV), num_steps=2, y=yd)  # one Euler step over [0, 1]: x + 1.0 * model(x, 0)
        v0 = m(x.to(DEV), torch.zeros(bs, device=DEV, dtype=torch.bfloat16), yd)
    assert torch.isfinite(out.float()).all() and torch.isfinite(step.float()).all()
    assert torch.equal(out[k:k + 1], one), f"{name}: batch row differs from its bs=1 run"
    check_close(step, (x.to(DEV).float() + v0.float()).bfloat16(), f"{name} whole-loop graph step vs forward", rtol=2e-2, atol=2e-2, scale_atol=False, max_strict_viol=1.0)
    sd16 = {kk: v.bfloat16().float() for kk, v in sd.items()}                # the oracle sees the bf16-rounded weights
    want = _oracle_forward(cfg, sd16, x[k:k + 1].float(), tt[k:k + 1].float(), None if y is None else y[k:k + 1])
    check_close(one, want, f"{name} full depth bf16 bs={bs} row {k} vs fp32 oracle", rtol=8e-2, atol=8e-2, scale_atol=False, max_strict_viol=1.0)


def test_has_text_video_bf16_copy_free_temporal_layers():
    """has_text on a factorised video scan in bf16 at a width that takes the hot-path kernels (D = 128): the spatial layers run on
    (b t) sequences and the temporal layers copy-free through the composite row tables; the cross-attention branch needs the
    mixer output un-permuted first (each layer's own table).  Against the fp32 oracle on the bf16-rounded weights."""
    from zigma_b200 import ZigMa
    cfg = dict(in_channels=4, embed_dim=128, depth=3, img_dim=8, patch_size=2, scan_type="zzvideo_sst", use_pe=2, video_frames=8, tpe=True,
               has_text=True, d_context=24, n_context_token=7)
    m = ZigMa(device=DEV, dtype=torch.bfloat16, **cfg).eval()
    sd = synth.synth_state_dict({k: tuple(v.shape) for k, v in m.state_dict().items()}, seed=0, dtype=torch.bfloat16)
    m.load_state_dict(sd)
    x, tt, y = model_io(cfg, 2)
    with torch.no_grad():
        out = m(x.to(DEV).bfloat16(), tt.to(DEV).bfloat16(), y.to(DEV).bfloat16())
    assert m._engine is not None, "ZigMa.forward did not take the engine"
    want = _oracle_forward(cfg, {k: v.float() for k, v in sd.items()}, x.bfloat16().float(), tt.bfloat16().float(), y.bfloat16().float())
    check_close(out, want, "has_text + video bf16 engine vs fp32 oracle", rtol=6e-2, atol=6e-2, scale_atol=False, max_strict_viol=1.0)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_has_text_blocks_on_the_engine(dtype):
    """has_text models (cross-attention branch, 6-way adaLN; SURVEY.md section 8f-3): the sampling engine -- mixer through
    the fused kernels, attention branch handed to the fused tail as the "mix" operand -- against the per-op block loop."""
    from zigma_b200 import ZigMa
    cfg = dict(img_dim=8, patch_size=1, in_channels=4, embed_dim=64, depth=3, scan_type="zigzagN8", num_classes=-1, has_text=True, d_context=24,
               use_pe=0, rms_norm=True, fused_add_norm=True, residual_in_fp32=True)
    torch.manual_seed(0)
    m = ZigMa(device=DEV, dtype=dtype, **cfg).eval()
    with torch.no_grad():
        for p in m.parameters():
            if p.requires_grad and p.abs().sum() == 0:      # adaLN-zero init would silence both branches
                p.normal_(0, 0.05)
    g = torch.Generator(device=DEV).manual_seed(1)
    x = torch.randn(3, 4, 8, 8, device=DEV, generator=g).to(dtype)
    t = torch.rand(3, device=DEV, generator=g).to(dtype)
    ctx_dim = m.y_embedder.in_features if hasattr(m.y_embedder, "in_features") else m.y_embedder[0].in_features
    y = torch.randn(3, 7, ctx_dim, device=DEV, generator=g).to(dtype)
    with torch.no_grad():
        ref = m.forward_autograd(x, t, y)
        out = m(x, t, y)
    assert m._engine is not None, "ZigMa.forward did not take the engine"
    if dtype == torch.float32:
        check_close(out, ref, "has_text engine vs block loop (fp32)", atol=2e-5)
    else:
        check_close(out, ref, "has_text engine vs block loop (bf16)", rtol=5e-2, atol=5e-2, max_strict_viol=1.0)
