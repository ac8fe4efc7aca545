"""GPU (H100): the text cross-attention kernels (zg_cross_attn_fwd / _bwd, zigma_b200/attention.py) against an fp64
reference built from the inputs as given (forward formula, fp64 autograd for the gradients).

Bounds, per element, with no blanket rtol:   |got - ref| <= C * u * S + 1 ulp(ref) of the output dtype
  (one ulp at least the dtype's smallest normal number, an absolute floor for results near the underflow threshold)
  u  the unit roundoff of the dtype P is rounded to: 2^-24 (fp32), 2^-11 (fp16), 2^-8 (bf16);
  S  the sum of |terms| forming the element, the score error amplified by the score magnitude  a_i = 1 + max_j |s_ij|:
       O_i      sum_j p_ij |v_j| a_i
       dV_j     sum_i p_ij |dO_i| a_i
       dQ_i     0.125 sum_j p_ij (|dP_ij| + |D_i|) |k_j| a_i
       dK_j     0.125 sum_i p_ij (|dP_ij| + |D_i|) |q_i| a_i
     (s = 0.125 q.k, p = softmax(s), dP = dO.v, D = dO.O, all fp64).
  C  fp32 64 (64-term fp32 dot products, MUFU exp2 with 2^-22 relative error, sums over up to 256 keys);
     fp16 / bf16 4 (P rounded once to the I/O dtype; the backward reads the rounded O).
The fraction of the bound each check reaches goes to $ZIGMA_PARITY_LOG.  Two checks keep the bound honest: it rejects the
forward with the largest-weight key dropped (CPU), and library SDPA meets it on the same inputs."""
import json
import os

import pytest
import torch
import torch.nn.functional as F

DEV = "cuda"
U = {torch.float32: 2.0 ** -24, torch.float16: 2.0 ** -11, torch.bfloat16: 2.0 ** -8}
C = {torch.float32: 64.0, torch.float16: 4.0, torch.bfloat16: 4.0}
H_DIM = 64
gpu = pytest.mark.gpu


def _mant(dtype):
    return {torch.float32: 23, torch.float16: 10, torch.bfloat16: 7}[dtype]


def _ulp(x, dtype):
    """One unit in the last place of |x| in `dtype`, 2^(floor(log2 |x|) - mantissa bits), but at least the smallest normal
    number: near the underflow threshold exp2 (and the terms it scales) lose relative precision, so gradients of order 1e-38
    in fp32 may be off by that much absolutely."""
    fi = torch.finfo(dtype)
    e = torch.floor(torch.log2(x.abs().clamp_min(fi.tiny)))
    return torch.exp2(e - _mant(dtype)).clamp_min(fi.tiny)


def _split(t, heads):
    B, L, _ = t.shape
    return t.reshape(B, L, heads, H_DIM).transpose(1, 2).double()          # (B, H, L, 64)


def _merge(t):
    B, H, L, _ = t.shape
    return t.transpose(1, 2).reshape(B, L, H * H_DIM)


def reference(q, k, v, heads, do=None):
    """fp64 forward (and gradients for dO = do) plus the bound sums S of every output (see the module docstring)."""
    qd, kd, vd = (_split(x.detach().cpu(), heads).requires_grad_(do is not None) for x in (q, k, v))
    s = (qd @ kd.transpose(-1, -2)) * 0.125
    p = s.softmax(-1)
    o = p @ vd
    amp = 1.0 + s.detach().abs().amax(-1, keepdim=True)                         # (B, H, L, 1)
    pa = p.detach() * amp
    out = {"o": _merge(o.detach()), "S_o": _merge(pa @ vd.detach().abs())}
    if do is not None:
        dod = _split(do.detach().cpu(), heads)
        o.backward(dod)
        dP = dod @ vd.detach().transpose(-1, -2)
        D = (dod * o.detach()).sum(-1, keepdim=True)
        w = pa * (dP.abs() + D.abs())
        out.update(dq=_merge(qd.grad), dk=_merge(kd.grad), dv=_merge(vd.grad),
                   S_dq=_merge(0.125 * w @ kd.detach().abs()), S_dk=_merge(0.125 * w.transpose(-1, -2) @ qd.detach().abs()),
                   S_dv=_merge(pa.transpose(-1, -2) @ dod.abs()))
    return out


def bound_fraction(got, ref, S, dtype):
    """max over elements of |got - ref| / (C u S + 1 ulp(ref)); <= 1 passes."""
    got = got.detach().double().cpu()
    lim = C[dtype] * U[dtype] * S + _ulp(ref, dtype)
    return ((got - ref).abs() / lim).max().item() if got.numel() else 0.0


def _log(what, frac):
    path = os.environ.get("ZIGMA_PARITY_LOG")
    if path:
        try:
            with open(path, "a") as f:
                f.write(json.dumps(dict(test=os.environ.get("PYTEST_CURRENT_TEST", "").split(" ")[0], what=what, bound_fraction=frac)) + "\n")
        except OSError:
            pass


def check(what, got, ref, S, dtype):
    frac = bound_fraction(got, ref, S, dtype)
    print(f"    {what}: {frac:.3f} of the bound")
    _log(what, frac)
    assert got.shape == ref.shape and torch.isfinite(got.float()).all(), what
    assert frac <= 1.0, f"{what}: error {frac:.3f} x the bound"


def inputs(B, L, Lk, heads, dtype, seed=0, fused=False, scale=1.0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    dim = heads * H_DIM
    if fused:      # q, k, v as column slices of one (rows, 3 dim) buffer
        buf = torch.randn(B, max(L, Lk), 3 * dim, device=DEV, generator=g).to(dtype)
        q, k, v = buf[:, :L, :dim], buf[:, :Lk, dim:2 * dim], buf[:, :Lk, 2 * dim:]
    else:
        q = (scale * torch.randn(B, L, dim, device=DEV, generator=g)).to(dtype)
        k = torch.randn(B, Lk, dim, device=DEV, generator=g).to(dtype)
        v = torch.randn(B, Lk, dim, device=DEV, generator=g).to(dtype)
    do = torch.randn(B, L, dim, device=DEV, generator=g).to(dtype)
    return q, k, v, do


def run(q, k, v, heads, do=None):
    from zigma_b200.attention import cross_attention_fn
    if do is None:
        with torch.no_grad():
            return {"o": cross_attention_fn(q, k, v, heads)}
    qr, kr, vr = (x.detach().requires_grad_() for x in (q, k, v))
    o = cross_attention_fn(qr, kr, vr, heads)
    o.backward(do)
    return {"o": o.detach(), "dq": qr.grad, "dk": kr.grad, "dv": vr.grad}


def check_all(tag, got, ref, dtype):
    for name in ("o", "dq", "dk", "dv"):
        if name in got:
            check(f"{tag} {name}", got[name], ref[name], ref["S_" + name].double(), dtype)


# ---- the bound is not vacuous (CPU) ----------------------------------------------------------------------------------
def test_forward_bound_rejects_a_dropped_key():
    """With the largest-weight key of one row dropped from the softmax, the forward misses the bound by far, in every dtype."""
    g = torch.Generator().manual_seed(3)
    for dtype in (torch.float32, torch.float16, torch.bfloat16):
        q, k, v = (torch.randn(2, 5, 128, generator=g).to(dtype) for _ in range(3))
        k, v = k[:, :7].contiguous(), v[:, :7].contiguous()
        ref = reference(q, k, v, 2)
        qd, kd, vd = _split(q, 2), _split(k, 2), _split(v, 2)
        s = (qd @ kd.transpose(-1, -2)) * 0.125
        j = s[0, 0, 0].argmax()
        s[0, 0, 0, j] = -float("inf")
        bad = _merge(s.softmax(-1) @ vd).to(dtype)
        assert bound_fraction(bad, ref["o"], ref["S_o"], dtype) > 10.0, dtype
        assert bound_fraction(ref["o"].to(dtype), ref["o"], ref["S_o"], dtype) <= 1.0


# ---- the case matrix -------------------------------------------------------------------------------------------------
DTYPES = [torch.float32, torch.float16, torch.bfloat16]
DT_ID = {torch.float32: "fp32", torch.float16: "fp16", torch.bfloat16: "bf16"}


@gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
@pytest.mark.parametrize("Lk", [1, 7, 16, 77, 128, 200, 256])
def test_keys(dtype, Lk):
    """Every key count class: one key, below one MMA tile, tile multiples, the CLIP context, one and several 64-key chunks."""
    q, k, v, do = inputs(3, 37, Lk, 8, dtype, seed=Lk)
    got, ref = run(q, k, v, 8, do), reference(q, k, v, 8, do)
    check_all(f"{DT_ID[dtype]} B3 L37 Lk{Lk} H8", got, ref, dtype)
    if Lk == 1:       # softmax over one key is 1: dS = 0, so dQ and dK are exactly zero
        assert not got["dq"].any() and not got["dk"].any()


@gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
@pytest.mark.parametrize("B,L,Lk,H", [(1, 1, 77, 1), (2, 1024, 77, 8), (1, 4096, 200, 1), (64, 37, 77, 8), (4, 1024, 256, 8)])
def test_shapes(dtype, B, L, Lk, H):
    q, k, v, do = inputs(B, L, Lk, H, dtype, seed=B * 7 + L)
    got, ref = run(q, k, v, H, do), reference(q, k, v, H, do)
    check_all(f"{DT_ID[dtype]} B{B} L{L} Lk{Lk} H{H}", got, ref, dtype)


@gpu
def test_sampling_shape_forward():
    """The sampling shape of the demo model: bs 64, 1024 tokens, 8 heads, 77 keys (forward only, bf16)."""
    q, k, v, _ = inputs(64, 1024, 77, 8, torch.bfloat16, seed=11)
    got = run(q, k, v, 8)
    sel = [0, 31, 63]
    ref = reference(q[sel], k[sel], v[sel], 8)
    check("bf16 B64 L1024 Lk77 forward (rows 0, 31, 63)", got["o"][sel], ref["o"], ref["S_o"], torch.bfloat16)


@gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
def test_fused_qkv_slices(dtype):
    """q, k, v as column slices of one (rows, 3 * 512) buffer: row stride 1536, no copies."""
    q, k, v, do = inputs(4, 100, 77, 8, dtype, seed=5, fused=True)
    assert q.stride(1) == 3 * 512 and not q.is_contiguous()
    got, ref = run(q, k, v, 8, do), reference(q, k, v, 8, do)
    check_all(f"{DT_ID[dtype]} fused qkv", got, ref, dtype)


@gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
@pytest.mark.parametrize("case", ["zeros", "equal_keys", "scores_1e3"])
def test_edge_inputs(dtype, case):
    """Zero inputs (uniform softmax), equal keys (uniform softmax, dQ = 0 up to rounding), and scores near +-1e3, which
    overflow exp without the max subtraction."""
    q, k, v, do = inputs(2, 64, 77, 8, dtype, seed=9)
    if case == "zeros":
        q, k = torch.zeros_like(q), torch.zeros_like(k)
    elif case == "equal_keys":
        k = k[:, :1].expand_as(k).contiguous()
    else:
        q = (q.float() * 250).to(dtype)           # |s| = |q.k| / 8 up to about 1e3
    got, ref = run(q, k, v, 8, do), reference(q, k, v, 8, do)
    if case == "scores_1e3":
        qd, kd = _split(q.cpu(), 8), _split(k.cpu(), 8)
        assert ((qd @ kd.transpose(-1, -2)) * 0.125).abs().max() > 500
    check_all(f"{DT_ID[dtype]} {case}", got, ref, dtype)


@gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
def test_library_sdpa_meets_the_bound(dtype):
    """The bound is not cut to fit the new kernel: PyTorch's SDPA on the same inputs meets it too (forward and gradients)."""
    q, k, v, do = inputs(2, 200, 77, 8, dtype, seed=21)
    qr, kr, vr = (x.detach().clone().requires_grad_() for x in (q, k, v))
    sp = lambda t: t.reshape(t.shape[0], t.shape[1], 8, H_DIM).transpose(1, 2)
    o = _merge(F.scaled_dot_product_attention(sp(qr), sp(kr), sp(vr)))
    o.backward(do)
    ref = reference(q, k, v, 8, do)
    check_all(f"{DT_ID[dtype]} SDPA", {"o": o.detach(), "dq": qr.grad, "dk": kr.grad, "dv": vr.grad}, ref, dtype)


@gpu
def test_misaligned_pointer_is_rejected():
    """A 16-bit q whose base pointer is 2 bytes off a 16-byte boundary is rejected with a RuntimeError (no fault, no copy)."""
    from zigma_b200.attention import cross_attention_fn
    buf = torch.randn(2, 8, 513, device=DEV).bfloat16()
    q = buf[:, :, 1:]                              # 2 bytes in
    k = torch.randn(2, 7, 512, device=DEV).bfloat16()
    with pytest.raises(RuntimeError, match="aligned"):
        cross_attention_fn(q, k, k, 8)
    with pytest.raises(RuntimeError, match="Lk"):
        cross_attention_fn(torch.randn(1, 4, 512, device=DEV), torch.randn(1, 257, 512, device=DEV), torch.randn(1, 257, 512, device=DEV), 8)


# ---- bitwise properties ----------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
def test_batch_row_equals_row_alone(dtype):
    q, k, v, do = inputs(5, 300, 77, 8, dtype, seed=2)
    full = run(q, k, v, 8, do)
    for r in (0, 3):
        one = run(q[r:r + 1], k[r:r + 1], v[r:r + 1], 8, do[r:r + 1])
        assert torch.equal(full["o"][r:r + 1], one["o"]) and torch.equal(full["dq"][r:r + 1], one["dq"]), (dtype, r)


@gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
def test_dk_dv_repeat_bitwise(dtype):
    """dK / dV are sums over all query rows: they repeat bit for bit idle, beside a concurrent matmul, and with the
    deterministic flag on and off (there are no atomics to order)."""
    q, k, v, do = inputs(16, 1024, 77, 8, dtype, seed=4)
    base = run(q, k, v, 8, do)
    a = torch.randn(4096, 4096, device=DEV)
    side = torch.cuda.Stream()
    prev = torch.are_deterministic_algorithms_enabled()
    try:
        for det in (False, True):
            torch.use_deterministic_algorithms(det)
            for busy in (False, True):
                if busy:
                    side.wait_stream(torch.cuda.current_stream())
                    with torch.cuda.stream(side):
                        for _ in range(8):
                            a = a @ a * 1e-2
                got = run(q, k, v, 8, do)
                for n in ("o", "dq", "dk", "dv"):
                    assert torch.equal(got[n], base[n]), (n, det, busy)
                torch.cuda.synchronize()
    finally:
        torch.use_deterministic_algorithms(prev)


def _text_model(dtype, embed_dim=64, d_context=24, depth=2, img_dim=8, patch_size=1, seed=0):
    from zigma_b200 import ZigMa
    torch.manual_seed(seed)
    m = ZigMa(in_channels=4, embed_dim=embed_dim, depth=depth, img_dim=img_dim, patch_size=patch_size, scan_type="zigzagN8",
              num_classes=-1, has_text=True, d_context=d_context, use_pe=2, device=DEV, dtype=dtype)
    with torch.no_grad():
        for p in m.parameters():
            if p.abs().sum() == 0:           # adaLN-zero init would silence the attention branch
                p.normal_(0, 0.05)
    return m.eval()


@gpu
def test_sample_euler_graph_replay_equals_eager_loop():
    """ZigMa.sample_euler on a has_text model (the whole loop as one CUDA-graph replay) equals the eager loop bit for bit."""
    from zigma_b200.engine import loop_eager
    m = _text_model(torch.bfloat16)
    g = torch.Generator(device=DEV).manual_seed(1)
    x0 = torch.randn(2, 4, 8, 8, device=DEV, generator=g).bfloat16()
    y = torch.randn(2, 77, 24, device=DEV, generator=g).bfloat16()
    with torch.no_grad():
        m.sample_euler(x0 * 0.5, num_steps=5, y=y)                 # capture
        got = m.sample_euler(x0, num_steps=5, y=y)                 # replay
        grid = torch.linspace(0.0, 1.0, 5)
        want = loop_eager(m._engine, x0, grid.tolist(), (grid[1:] - grid[:-1]).tolist(), y, False)
    assert torch.equal(got, want)


# ---- model level -----------------------------------------------------------------------------------------------------
@gpu
def test_demo_width_model_bf16_vs_oracle():
    """The reference's demo has_text width (D 768, 77 CLIP tokens of width 768), 32 x 32 latents, patch 1, depth 2: bf16 on
    the engine against the fp32 oracle on the bf16-rounded weights, at test_gpu_model.py's whole-model bf16 tolerance."""
    from oracle import synth, zigma_oracle as zo
    from util import check_close
    from zigma_b200 import ZigMa
    cfg = dict(in_channels=4, embed_dim=768, depth=2, img_dim=32, patch_size=1, scan_type="zigzagN8", use_pe=2, has_text=True,
               d_context=768, n_context_token=77)
    m = ZigMa(device=DEV, dtype=torch.bfloat16, **cfg).eval()
    sd = synth.synth_state_dict({k: tuple(v.shape) for k, v in m.state_dict().items()}, seed=0, dtype=torch.bfloat16)
    m.load_state_dict(sd)
    g = torch.Generator().manual_seed(6)
    x, tt, y = torch.randn(1, 4, 32, 32, generator=g), torch.rand(1, generator=g), torch.randn(1, 77, 768, generator=g)
    with torch.no_grad():
        out = m(x.to(DEV).bfloat16(), tt.to(DEV).bfloat16(), y.to(DEV).bfloat16())
    assert m._engine is not None
    zo.USE_C_SCAN = True
    try:
        want = zo.zigma_forward({k: v.float() for k, v in sd.items()}, dict(cfg, norm_epsilon=1e-5), x.bfloat16().float(),
                                tt.bfloat16().float(), y.bfloat16().float())
    finally:
        zo.USE_C_SCAN = False
    check_close(out, want, "demo-width has_text bf16 engine vs fp32 oracle", rtol=6e-2, atol=6e-2, scale_atol=False, max_strict_viol=1.0)


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


@gpu
def test_profiler_kernels_per_block():
    """The engine forward launches the new forward kernel once per block and no ATen attention kernel; a training step
    launches the backward (dQ, dK / dV, segment reduction) once per block."""
    depth = 3
    m = _text_model(torch.bfloat16, embed_dim=128, depth=depth)
    g = torch.Generator(device=DEV).manual_seed(2)
    x = torch.randn(2, 4, 8, 8, device=DEV, generator=g).bfloat16()
    t = torch.rand(2, device=DEV, generator=g).bfloat16()
    y = torch.randn(2, 77, 24, device=DEV, generator=g).bfloat16()
    with torch.no_grad():
        m(x, t, y)
    os.environ["ZIGMA_CUDA_GRAPH"] = "0"
    try:
        with torch.no_grad():
            c = _kernel_counts(lambda: m(x, t, y))
    finally:
        del os.environ["ZIGMA_CUDA_GRAPH"]
    fwd = sum(n for k, n in c.items() if "xattn_fwd_mma_kernel" in k)
    aten = [k for k in c if any(s in k.lower() for s in ("fmha", "flash", "attention", "softmax"))]
    assert fwd == depth and not aten, (fwd, aten)
    m.train()
    c = _kernel_counts(lambda: m.forward_autograd(x, t, y).float().square().mean().backward())
    per = {s: sum(n for k, n in c.items() if s in k) for s in ("xattn_rows_kernel", "xattn_bwd_kv_kernel", "xattn_bwd_reduce_kernel",
                                                               "xattn_fwd_mma_kernel")}
    assert all(n == depth for n in per.values()), per
    assert not [k for k in c if any(s in k.lower() for s in ("fmha", "flash", "attention"))]


# ---- determinism of whole training steps -----------------------------------------------------------------------------
@gpu
def test_has_text_training_steps_repeat_bitwise():
    """tests/_xattn_det_worker.py in two fresh processes: the digests of 3 train_steps of two has_text configs, fp32 / bf16
    autocast / bf16 parameters, are equal."""
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    worker = os.path.join(root, "tests", "_xattn_det_worker.py")
    runs = []
    for _ in range(2):
        r = subprocess.run([sys.executable, worker], capture_output=True, text=True, timeout=1800, cwd=root)
        assert r.returncode == 0 and "XATTN_DET_WORKER_OK" in r.stdout, r.stdout[-3000:] + r.stderr[-6000:]
        runs.append([l for l in r.stdout.splitlines() if l.startswith("DIGEST ")])
    assert len(runs[0]) >= 6
    diff = [(a, b) for a, b in zip(*runs) if a != b]
    assert len(runs[0]) == len(runs[1]) and not diff, diff[:10]
