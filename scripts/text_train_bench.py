"""The text prologue of has_text blocks (zg_text_prologue_fwd / _bwd): what it costs against the eager chain it replaces, and
what it does to sampling and training of a text-conditioned model at the demo width.

    python scripts/text_train_bench.py [--reps 7] [--out results.json]

Demo width: D 768, depth 24, 32 x 32 latents, patch 1 (L 1024), 77 text tokens of width 768, bf16.
1. The prologue alone against the eager chain it replaces (index_select un-permutation, gated add, no-affine LayerNorm,
   modulate): forward at bs 64 (sampling), forward + backward at bs 16 (training), random zigzag row table.
2. One engine forward at bs 64 with eager launches (no CUDA graph).
3. One training step (forward + MSE backward, as scripts/droppath_bench.py times it; train mode, drop_path_rate 0.1) at
   bs 16 on the fused loop (ZIGMA_FUSED_TRAIN_TAIL=1) vs the per-op block loop (=0), bf16 weights; and the agreement of the
   two on one seed at that size.
4. The HBM roofline of the forward: bytes from the shapes (read x and mix, write hidden and q_in) over the data-sheet
   3.35 TB/s of the H100 SXM, against the measured kernel time.

Variants are alternated within each repetition; medians with min-max over the repetitions.  The card name and its power
limit are read in the same run and printed with the numbers."""
import argparse
import json
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

from zigma_b200 import ZigMa, _lib, synth  # noqa: E402
from zigma_b200.block_ops import text_prologue_fn  # noqa: E402

DEV = "cuda"
L, D, CTX = 1024, 768, 77
HBM_TBS = 3.35          # H100 SXM data sheet


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError, IndexError):
        q = "unknown"
    return {"gpu": name, "power_limit_and_max_sm_clock": q}


def events_ms(fn, n):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(n):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / n


def summary(xs):
    return {"median": statistics.median(xs), "min": min(xs), "max": max(xs), "n": len(xs)}


def alternate(variants, reps, n, warm=3):
    for fn in variants.values():
        for _ in range(warm):
            fn()
    torch.cuda.synchronize()
    t = {k: [] for k in variants}
    for _ in range(reps):
        for k, fn in variants.items():
            t[k].append(events_ms(fn, n))
    return {k: summary(v) for k, v in t.items()}


def eager_chain(x, mix, rowmap64, gate, shift, scale):
    """The engine's text branch before the prologue kernel: un-permute, gated add, norm_msa, modulate."""
    hidden = x + gate.unsqueeze(1) * mix.index_select(1, rowmap64)
    return hidden, F.layer_norm(hidden, (x.shape[-1],), eps=1e-6) * (1 + scale.unsqueeze(1)) + shift.unsqueeze(1)


def _operands(B, requires_grad=False):
    g = torch.Generator(device=DEV).manual_seed(0)
    rn = lambda *s: torch.randn(*s, device=DEV, generator=g).bfloat16()
    x, mix = rn(B, L, D), rn(B, L, D)
    mods = 0.3 * rn(B, 6 * D)
    perm = torch.randperm(L, device=DEV, generator=g)
    if requires_grad:
        x, mix, mods = x.requires_grad_(), mix.requires_grad_(), mods.requires_grad_()
    return x, mix, mods, perm


# ------------------------------------------------------------------------------------------------ 1./4. the prologue alone
def prologue(reps):
    out = {"unit": "us per call"}
    B = 64
    x, mix, mods, perm = _operands(B)
    gate, shift, scale = mods[:, 2 * D:3 * D], mods[:, 3 * D:4 * D], mods[:, 4 * D:5 * D]
    rowmap = perm.to(torch.int32)
    hidden, q_in = torch.empty_like(x), torch.empty_like(x)
    p = _lib.TextPrologueParams()
    p.x, p.mix, p.gate, p.shift, p.scale, p.rowmap = (_lib.ptr(t) for t in (x, mix, gate, shift, scale, rowmap))
    p.hidden, p.q_in, p.mod_rs = _lib.ptr(hidden), _lib.ptr(q_in), 6 * D
    p.batch, p.seqlen, p.dim, p.dtype, p.eps = B, L, D, _lib.ZG_BF16, 1e-6
    fwd = alternate({"kernel_fwd": lambda: _lib.call("zg_text_prologue_fwd", p),
                     "eager_fwd": lambda: eager_chain(x, mix, perm, gate, shift, scale)}, reps, 20)
    out["sampling_bs64"] = {k: {kk: (vv * 1e3 if kk != "n" else vv) for kk, vv in v.items()} for k, v in fwd.items()}
    out["sampling_bs64"]["eager_over_kernel"] = fwd["eager_fwd"]["median"] / fwd["kernel_fwd"]["median"]
    with torch.no_grad():
        e_h, e_q = eager_chain(x, mix, perm, gate, shift, scale)
    _lib.call("zg_text_prologue_fwd", p)
    out["sampling_bs64"]["max_abs_diff_vs_eager"] = {"hidden": (hidden.float() - e_h.float()).abs().max().item(),
                                                     "q_in": (q_in.float() - e_q.float()).abs().max().item()}
    nbytes = 4 * B * L * D * 2 + 3 * B * D * 2
    floor_us = nbytes / (HBM_TBS * 1e12) * 1e6
    out["roofline_bs64"] = {"bytes": nbytes, "hbm_floor_us_at_3.35TBs": floor_us,
                            "measured_us": fwd["kernel_fwd"]["median"] * 1e3,
                            "achieved_TBs": nbytes / (fwd["kernel_fwd"]["median"] * 1e-3) / 1e12,
                            "fraction_of_datasheet_bw": floor_us / (fwd["kernel_fwd"]["median"] * 1e3)}
    del x, mix, hidden, q_in
    torch.cuda.empty_cache()

    B = 16
    x, mix, mods, perm = _operands(B, requires_grad=True)
    rowmap = perm.to(torch.int32)
    g = torch.Generator(device=DEV).manual_seed(1)
    d_h, d_q = torch.randn(B, L, D, device=DEV, generator=g).bfloat16(), torch.randn(B, L, D, device=DEV, generator=g).bfloat16()

    def fused():
        c = mods.chunk(6, dim=1)
        h, q = text_prologue_fn(x, mix, c[2], rowmap, c[3], c[4], 1e-6)
        torch.autograd.backward([h, q], [d_h, d_q])

    def eager():
        c = mods.chunk(6, dim=1)
        h, q = eager_chain(x, mix, perm, c[2], c[3], c[4])
        torch.autograd.backward([h, q], [d_h, d_q])
    tr = alternate({"kernel_fwd_bwd": fused, "eager_fwd_bwd": eager}, reps, 10)
    out["training_bs16"] = {k: {kk: (vv * 1e3 if kk != "n" else vv) for kk, vv in v.items()} for k, v in tr.items()}
    out["training_bs16"]["eager_over_kernel"] = tr["eager_fwd_bwd"]["median"] / tr["kernel_fwd_bwd"]["median"]
    return out


# ------------------------------------------------------------------------------------------------ 2./3. model level
CFG = dict(img_dim=32, patch_size=1, in_channels=4, embed_dim=D, depth=24, scan_type="zigzagN8", num_classes=-1, use_pe=2,
           has_text=True, d_context=768, n_context_token=CTX, drop_path_rate=0.1)


def _model():
    m = ZigMa(device=DEV, dtype=torch.bfloat16, **CFG)
    m.load_state_dict(synth.synth_state_dict({k: tuple(v.shape) for k, v in m.state_dict().items()}, seed=0, dtype=torch.bfloat16))
    return m


def engine(reps, m, bs=64):
    g = torch.Generator(device=DEV).manual_seed(2)
    x = torch.randn(bs, 4, 32, 32, device=DEV, generator=g).bfloat16()
    t = torch.rand(bs, device=DEV, generator=g).bfloat16()
    y = torch.randn(bs, CTX, 768, device=DEV, generator=g).bfloat16()
    m.eval()
    os.environ["ZIGMA_CUDA_GRAPH"] = "0"
    try:
        with torch.no_grad():
            r = alternate({"engine_forward": lambda: m(x, t, y)}, reps, 2, warm=2)
    finally:
        os.environ.pop("ZIGMA_CUDA_GRAPH", None)
    return {"bs": bs, "unit": "ms per forward, eager launches", **r}


def steps(reps, m, bs=16):
    g = torch.Generator(device=DEV).manual_seed(1)
    x = torch.randn(bs, 4, 32, 32, device=DEV, generator=g).bfloat16()
    t = torch.rand(bs, device=DEV, generator=g).bfloat16()
    y = torch.randn(bs, CTX, 768, device=DEV, generator=g).bfloat16()
    target = torch.randn(bs, 4, 32, 32, device=DEV, generator=g).float()

    def step(fused, seed=None):
        def run():
            os.environ["ZIGMA_FUSED_TRAIN_TAIL"] = "1" if fused else "0"
            m.train()
            if seed is not None:
                torch.manual_seed(seed)
            for p_ in m.parameters():
                p_.grad = None
            out = m.forward_autograd(x, t, y)
            ((out.float() - target) ** 2).mean().backward()
            return out
        return run
    try:
        r = alternate({"train_fused": step(True), "train_per_op": step(False)}, reps, 3, warm=2)
        r["unit"] = "ms per forward + backward, bs %d, bf16 weights, train mode" % bs
        r["per_op_over_fused"] = r["train_per_op"]["median"] / r["train_fused"]["median"]
        outs, grads, rng = {}, {}, {}
        for fused in (True, False):
            o = step(fused, seed=1234)()
            outs[fused] = o.detach().float()
            rng[fused] = torch.cuda.get_rng_state()
            grads[fused] = {k: v.grad.float().clone() for k, v in m.named_parameters() if v.grad is not None}
        r["same_generator_state"] = bool(torch.equal(rng[True], rng[False]))
        r["out_max_abs_diff"], r["out_max_abs"] = (outs[True] - outs[False]).abs().max().item(), outs[False].abs().max().item()
        r["grad_worst_rel_l2"] = max(((grads[True][k] - grads[False][k]).norm() / (grads[False][k].norm() + 1e-30)).item()
                                     for k in grads[False])
    finally:
        os.environ.pop("ZIGMA_FUSED_TRAIN_TAIL", None)
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("text_train_bench: needs a CUDA device")
    r = {"card": card(), "prologue": prologue(a.reps)}
    m = _model()
    r["engine"] = engine(a.reps, m)
    r["train_step"] = steps(a.reps, m)
    print(json.dumps(r, indent=1))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(r, f, indent=1)


if __name__ == "__main__":
    main()
