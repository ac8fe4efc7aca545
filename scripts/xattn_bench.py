"""Cross-attention timings on the GPU (CUDA events): the zg_cross_attn kernels against library SDPA at the shapes of the
reference's text-conditioned demo model (D 768, 8 heads x 64, 77 CLIP tokens), in bf16.

    python scripts/xattn_bench.py [--reps 7] [--iters 50] [--depth 24] [--skip-engine]

  op        sampling: forward, B 64, L 1024, H 8, Lk 77;  training: forward + backward, B 16
  module    to_q .. to_out of one CrossAttention, the kernel path against the SDPA path with its (B, H, L, 64) reshapes and the
            transpose-and-copy before to_out, alternated call by call
  engine    one sampling-engine forward of the demo-width has_text model at depth 24, bs 64, eager (no graph), with the attention
            on the kernel and on SDPA, alternated

Each line gives the median and the min..max over --reps repeats of --iters calls.  The card's name and power limit are
printed by the same run.  The forward's roofline is HBM: Q read + O written (K, V are 77 rows per batch element)."""
import argparse
import os
import statistics
import subprocess
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

HBM = 3.35e12          # H100 SXM data sheet, bytes / s
MMA = 989e12           # dense BF16 FLOP / s


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name()


def timed(fn, iters):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / iters * 1e3     # us per call


def compare(label, fns, reps, iters):
    """fns: {name: callable}; warmed up, then timed alternately rep by rep."""
    for f in fns.values():
        for _ in range(3):
            f()
    torch.cuda.synchronize()
    res = {n: [] for n in fns}
    for _ in range(reps):
        for n, f in fns.items():
            res[n].append(timed(f, iters))
    for n, v in res.items():
        print(f"{label:10s} {n:34s} median {statistics.median(v):9.1f} us   [{min(v):.1f} .. {max(v):.1f}]", flush=True)
    return {n: statistics.median(v) for n, v in res.items()}


def sdpa(q, k, v, heads):
    B, L, dim = q.shape
    sp = lambda t: t.reshape(B, t.shape[1], heads, -1).transpose(1, 2)
    return F.scaled_dot_product_attention(sp(q), sp(k), sp(v)).transpose(1, 2).reshape(B, L, dim)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--depth", type=int, default=24)
    ap.add_argument("--skip-engine", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("xattn_bench: needs a CUDA device")
    from zigma_b200 import model_zigma
    from zigma_b200.attention import cross_attention_fn
    print(f"card: {card()}", flush=True)
    dev, dt, H, Lk, L = "cuda", torch.bfloat16, 8, 77, 1024
    g = torch.Generator(device=dev).manual_seed(0)

    # ---- op level -----------------------------------------------------------------------------------------------------
    B = 64
    q = torch.randn(B, L, H * 64, device=dev, generator=g, dtype=dt)
    k = torch.randn(B, Lk, H * 64, device=dev, generator=g, dtype=dt)
    v = torch.randn(B, Lk, H * 64, device=dev, generator=g, dtype=dt)
    with torch.no_grad():
        t = compare("op fwd", {"kernel B64": lambda: cross_attention_fn(q, k, v, H), "sdpa (+copy) B64": lambda: sdpa(q, k, v, H)},
                    a.reps, a.iters)
    nbytes = 2 * q.numel() * 2 + 2 * k.numel() * 2
    flops = 2 * 2 * B * H * L * Lk * 64
    floor = max(nbytes / HBM, flops / MMA) * 1e6
    print(f"op fwd     roofline: {nbytes / 1e6:.0f} MB -> {nbytes / HBM * 1e6:.1f} us at 3.35 TB/s; {flops / 1e9:.1f} GFLOP -> "
          f"{flops / MMA * 1e6:.1f} us at 989 TFLOP/s; kernel at {floor / t['kernel B64']:.0%} of the HBM bound", flush=True)

    B = 16
    qt, kt, vt = (x[:B].clone().requires_grad_() for x in (q, k, v))
    do = torch.randn(B, L, H * 64, device=dev, generator=g, dtype=dt)

    def train(fn):
        def f():
            o = fn(qt, kt, vt, H)
            torch.autograd.grad(o, (qt, kt, vt), do)
        return f
    compare("op f+b", {"kernel B16": train(cross_attention_fn), "sdpa (+copy) B16": train(sdpa)}, a.reps, a.iters)

    # ---- module level -------------------------------------------------------------------------------------------------
    D = 768
    attn = model_zigma.CrossAttention(D, D, heads=H).to(dev, dt).eval()
    x = torch.randn(64, L, D, device=dev, generator=g, dtype=dt)
    text = torch.randn(64, Lk, D, device=dev, generator=g, dtype=dt)

    def mod_sdpa():
        return attn.to_out(sdpa(attn.to_q(x), attn.to_k(text), attn.to_v(text), H))
    with torch.no_grad():
        compare("module", {"kernel B64": lambda: attn(x, text), "sdpa (+copies) B64": mod_sdpa}, a.reps, a.iters)

    # ---- one engine step of the demo-width model -----------------------------------------------------------------------
    if a.skip_engine:
        return
    from zigma_b200 import ZigMa
    from zigma_b200.engine import ZigMaEngine
    m = ZigMa(in_channels=4, embed_dim=D, depth=a.depth, img_dim=32, patch_size=1, scan_type="zigzagN8", use_pe=2, has_text=True,
              d_context=768, n_context_token=77, device=dev, dtype=dt).eval()
    eng = ZigMaEngine(m)
    xl = torch.randn(64, 4, 32, 32, device=dev, generator=g, dtype=dt)
    tt = torch.rand(64, device=dev, generator=g).to(dt)
    y = torch.randn(64, Lk, 768, device=dev, generator=g, dtype=dt)
    keys = model_zigma.MAX_KEYS

    def step(limit):
        def f():
            model_zigma.MAX_KEYS = limit        # 0 sends every CrossAttention call to the SDPA line
            try:
                eng._forward_impl(xl, tt, y)
            finally:
                model_zigma.MAX_KEYS = keys
        return f
    with torch.no_grad():
        compare(f"engine", {f"kernel depth {a.depth} bs 64": step(keys), f"sdpa depth {a.depth} bs 64": step(0)}, a.reps,
                max(1, a.iters // 10))


if __name__ == "__main__":
    main()
