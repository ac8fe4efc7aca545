"""Cost of PyTorch's deterministic mode for this package: the config-2 training step (D 640, depth 18, 32x32 latents, bs 16;
forward + backward) and each backward kernel alone at its layer shape, with torch.use_deterministic_algorithms off and on,
alternated, CUDA events.  Prints one JSON line.

    python scripts/det_bench.py [--bs 16] [--repeats 7] [--depth 18]

The step is timed with fp32 parameters under bf16 autocast ("amp") and with bf16 parameters ("bf16").  CUBLAS_WORKSPACE_CONFIG
is set for both settings (cuBLAS needs it under the flag), so the two differ only by the flag.  Times are medians over the
repeats, with min and max; "workspace_bytes" is the partials workspace of one call of each op."""
import argparse
import json
import os
import statistics
import subprocess
import sys

os.environ.setdefault("CUBLAS_WORKSPACE_CONFIG", ":4096:8")
import torch  # noqa: E402

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from zigma_b200 import ZigMa, _lib, synth  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--bs", type=int, default=16)
ap.add_argument("--repeats", type=int, default=7)
ap.add_argument("--depth", type=int, default=18)
args = ap.parse_args()
dev = "cuda"
D, E, L, N = 640, 1280, 1024, 16


def timed(fn, det, n):
    torch.use_deterministic_algorithms(det)
    try:
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        a.record()
        for _ in range(n):
            fn()
        b.record()
        torch.cuda.synchronize()
    finally:
        torch.use_deterministic_algorithms(False)
    return a.elapsed_time(b) / n


def compare(fn, repeats, inner):
    for det in (False, True, False, True):           # warm-up: modules, allocator, cuBLAS algorithms of both settings
        timed(fn, det, 1)
    off, on = [], []
    for _ in range(repeats):
        off.append(timed(fn, False, inner))
        on.append(timed(fn, True, inner))
    s = lambda v: {"median": round(statistics.median(v), 4), "min": round(min(v), 4), "max": round(max(v), 4)}
    return {"off_ms": s(off), "on_ms": s(on), "overhead_pct": round(100 * (statistics.median(on) / statistics.median(off) - 1), 2)}


res = {"bs": args.bs, "depth": args.depth, "repeats": args.repeats, "device": torch.cuda.get_device_name(0),
       "sms": torch.cuda.get_device_properties(0).multi_processor_count}
try:
    q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True, timeout=30).stdout.strip()
    res["power_limit_and_max_sm_clock"] = q
except Exception as e:      # (reported, not fatal: the timings stand without it)
    res["power_limit_and_max_sm_clock"] = f"unavailable: {e}"

# ---- whole training step (forward + backward), as scripts/train_bench.py runs it ----
CFG = dict(img_dim=32, patch_size=1, in_channels=4, embed_dim=D, depth=args.depth, scan_type="zigzagN8", num_classes=-1,
           has_text=False, use_pe=0, rms_norm=True, fused_add_norm=True, residual_in_fp32=True)
res["step"] = {}
for mode in ("amp", "bf16"):
    dtype = torch.bfloat16 if mode == "bf16" else torch.float32
    m = ZigMa(device=dev, dtype=dtype, **CFG)
    m.load_state_dict(synth.synth_state_dict({k: tuple(v.shape) for k, v in m.state_dict().items()}, seed=0, dtype=dtype))
    m.eval()
    g = torch.Generator(device=dev).manual_seed(1)
    x = torch.randn(args.bs, 4, 32, 32, device=dev, generator=g).to(dtype)
    tt = torch.rand(args.bs, device=dev, generator=g).to(dtype)
    target = torch.randn(args.bs, 4, 32, 32, device=dev, generator=g)

    def step():
        for p in m.parameters():
            p.grad = None
        with torch.autocast("cuda", dtype=torch.bfloat16, enabled=(mode == "amp")):
            out = m.forward_autograd(x, tt, None)
        ((out.float() - target) ** 2).mean().backward()
    res["step"][mode] = compare(step, args.repeats, 3)
    del m
    torch.cuda.empty_cache()

# ---- each backward op alone at the config-2 layer shape (bf16 activations, token-major) ----
from zigma_b200.selective_scan_interface import _scan_bwd, _scan_fwd  # noqa: E402
from zigma_b200.causal_conv1d_interface import _conv_bwd  # noqa: E402
from zigma_b200.layernorm import _norm_bwd, _norm_fwd  # noqa: E402
from zigma_b200.block_ops import block_tail_fn  # noqa: E402

g = torch.Generator(device=dev).manual_seed(2)
bs = args.bs
tok = lambda c, dt=torch.bfloat16: torch.randn(bs, L, c, device=dev, generator=g).to(dt)
ops, ws = {}, {}

u, z, dout = tok(E).transpose(1, 2), tok(E).transpose(1, 2), tok(E).transpose(1, 2)
delta = (0.5 * torch.rand(bs, L, E, device=dev, generator=g)).bfloat16().transpose(1, 2)
xbc = tok(2 * N)
B, C = xbc[:, :, :N].permute(0, 2, 1).unsqueeze(1), xbc[:, :, N:].permute(0, 2, 1).unsqueeze(1)
A = -0.5 * torch.rand(E, N, device=dev, generator=g)
Dv, bias = torch.randn(E, device=dev, generator=g), 0.5 * torch.rand(E, device=dev, generator=g)
rowmap = torch.randperm(L, device=dev, generator=g).to(torch.int32)
_, _, ckpt, saved = _scan_fwd(u, delta, A, B, C, Dv, z, bias, True, z_rowmap=rowmap, want_last_state=False, want_ckpt=True)
ops["scan_bwd"] = lambda: _scan_bwd(saved, ckpt, dout, True, z_rowmap=rowmap)

xc = tok(2 * E)[:, :, :E].transpose(1, 2)          # the conv half of in_proj's output
cw, cb = torch.randn(E, 4, device=dev, generator=g), torch.randn(E, device=dev, generator=g)
dconv = tok(E).transpose(1, 2)
ops["conv_bwd"] = lambda: _conv_bwd(xc, cw, cb, dconv, True, x_rowmap=rowmap)

xn, rn = tok(D).reshape(-1, D), torch.randn(bs * L, D, device=dev, generator=g)
nw = torch.ones(D, device=dev)
yn, mean, rstd, resout = _norm_fwd(xn, nw, None, 1e-5, rn, torch.float32, True)
dyn = tok(D).reshape(-1, D)
ops["add_norm_bwd"] = lambda: _norm_bwd(dyn, resout, nw, None, mean, rstd, None, True, True, torch.bfloat16)

bx, bmix = tok(D).requires_grad_(), tok(D).requires_grad_()
ada = torch.randn(bs, 3 * D, device=dev, generator=g).bfloat16().requires_grad_()
bres = torch.randn(bs, L, D, device=dev, generator=g).requires_grad_()
bnw = torch.ones(D, device=dev, dtype=torch.bfloat16).requires_grad_()
gate, shift, scale = ada.chunk(3, dim=1)
touts = block_tail_fn(bx, bmix, gate, shift, scale, bnw, bres, rowmap, 1e-5)
tgrads = (torch.randn(bs, L, D, device=dev, generator=g), tok(D), tok(D))
ops["block_tail_bwd"] = lambda: torch.autograd.grad(touts, (bx, bmix, ada, bnw, bres), tgrads, retain_graph=True)

res["ops"] = {k: compare(f, args.repeats, 20) for k, f in ops.items()}


# workspace bytes of one call, captured from the size queries the calls make
def capture_ws(fn):
    seen, orig = [], _lib.det_workspace_bytes

    def spy(name, params):
        n = orig(name, params)
        seen.append((name, n))
        return n
    _lib.det_workspace_bytes = spy
    try:
        timed(fn, True, 1)
    finally:
        _lib.det_workspace_bytes = orig
    return {name: n for name, n in seen}


res["workspace_bytes"] = {k: capture_ws(f) for k, f in ops.items()}
print(json.dumps(res))
