"""Stochastic depth on the fused block tail: what it costs, and what train mode gains from it.

    python scripts/droppath_bench.py [--reps 7] [--out results.json]

1. Kernels alone at the config-2 layer shape (bs 16, L 1024, D 640, bf16): zg_block_tail_fwd_dp vs zg_block_tail_fwd and
   zg_block_tail_bwd_dp vs zg_block_tail_bwd, the backward with torch.use_deterministic_algorithms off and on.
2. One training step (forward + MSE backward, as scripts/train_bench.py times it) of a config-2-width model (D 640, depth 18,
   bs 16, drop_path_rate 0.1): train mode on the fused tails vs train mode on the per-op block loop (ZIGMA_FUSED_TRAIN_TAIL=0),
   with the eval-mode step (fused, no drop path) as the reference point; fp32 weights under bf16 autocast, and bf16 weights.
3. The fused and the per-op train-mode step on the same seed: output and gradient agreement at the timed size.

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

from zigma_b200 import ZigMa, _lib, synth  # noqa: E402
from zigma_b200.block_ops import tail_bwd_nparts  # noqa: E402

DEV = "cuda"


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


# ------------------------------------------------------------------------------------------------ 1. kernels alone
def kernels(reps):
    B, L, D, T = 16, 1024, 640, torch.bfloat16
    g = torch.Generator(device=DEV).manual_seed(0)
    rn = lambda *s, dt=T: torch.randn(*s, device=DEV, generator=g).to(dt)
    x, mix, res = rn(B, L, D), rn(B, L, D), rn(B, L, D, dt=torch.float32)
    mods = rn(B, 3 * D) * 0.3
    shift, scale, gate = mods[:, :D], mods[:, D:2 * D], mods[:, 2 * D:]
    nw = 1 + 0.2 * rn(D)
    rowmap = torch.randperm(L, device=DEV, generator=g).to(torch.int32)
    ps = (torch.tensor([0, 1] * (B // 2), device=DEV).to(T) * torch.tensor(1.0, dtype=T).div_(0.9).to(DEV))
    res_out, normed, modded = torch.empty(B, L, D, device=DEV), torch.empty_like(x), torch.empty_like(x)
    rstd = torch.empty(B * L, device=DEV)
    p = _lib.BlockTailParams()
    p.x, p.mix, p.gate, p.shift, p.scale, p.norm_w = (_lib.ptr(t) for t in (x, mix, gate, shift, scale, nw))
    p.residual, p.rowmap, p.residual_out, p.normed, p.modded, p.rstd = (_lib.ptr(t) for t in (res, rowmap, res_out, normed, modded, rstd))
    p.mod_rs, p.batch, p.seqlen, p.dim, p.dtype, p.final_layer, p.eps = 3 * D, B, L, D, _lib.ZG_BF16, 0, 1e-5
    pdp = _lib.BlockTailDpParams(p, _lib.ptr(ps))
    nparts = tail_bwd_nparts(B, L, torch.cuda.get_device_properties(0).multi_processor_count)
    d_ro, d_n, d_m = rn(B, L, D, dt=torch.float32), rn(B, L, D), rn(B, L, D)
    d_x, d_mix, d_ri = torch.empty_like(x), torch.empty_like(x), torch.empty(B, L, D, device=DEV)
    acc, d_w = torch.zeros(3, B, D, device=DEV), torch.empty(nparts, D, device=DEV)
    q = _lib.BlockTailBwdParams()
    q.d_residual_out, q.d_normed, q.d_modded, q.r, q.rstd = (_lib.ptr(t) for t in (d_ro, d_n, d_m, res_out, rstd))
    q.mix, q.gate, q.scale, q.norm_w, q.rowmap = (_lib.ptr(t) for t in (mix, gate, scale, nw, rowmap))
    q.d_x, q.d_mix, q.d_residual_in, q.dgate, q.dshift, q.dscale, q.d_norm_w = (_lib.ptr(t) for t in (d_x, d_mix, d_ri, acc[0], acc[1], acc[2], d_w))
    q.mod_rs, q.batch, q.seqlen, q.dim, q.dtype, q.nparts = 3 * D, B, L, D, _lib.ZG_BF16, nparts
    qdp = _lib.BlockTailBwdDpParams(q, _lib.ptr(ps))
    out = {"shape": "bs 16 x L 1024 x D 640, bf16, rowmap, every operand", "unit": "us per call"}
    fwd = alternate({"plain_fwd": lambda: _lib.call("zg_block_tail_fwd", p), "dp_fwd": lambda: _lib.call("zg_block_tail_fwd_dp", pdp)},
                    reps, 50)
    for det in (False, True):
        torch.use_deterministic_algorithms(det)
        try:
            bwd = alternate({"plain_bwd": lambda: _lib.call_bwd("zg_block_tail_bwd", q),
                             "dp_bwd": lambda: _lib.call_bwd("zg_block_tail_bwd_dp", qdp)}, reps, 50)
        finally:
            torch.use_deterministic_algorithms(False)
        for k, v in bwd.items():
            fwd[f"{k}_det_{'on' if det else 'off'}"] = v
    for k, v in fwd.items():
        out[k] = {kk: (vv * 1e3 if kk != "n" else vv) for kk, vv in v.items()}
    return out


# ------------------------------------------------------------------------------------------------ 2./3. training step
CFG = dict(img_dim=32, patch_size=1, in_channels=4, embed_dim=640, depth=18, scan_type="zigzagN8", num_classes=-1, use_pe=0,
           drop_path_rate=0.1)


def steps(reps, bs=16):
    res = {}
    for label, dtype, amp in (("fp32_weights_bf16_autocast", torch.float32, True), ("bf16_weights", torch.bfloat16, False)):
        m = ZigMa(device=DEV, dtype=dtype, **CFG)
        m.load_state_dict(synth.synth_state_dict({k: tuple(v.shape) for k, v in m.state_dict().items()}, seed=0, dtype=dtype))
        g = torch.Generator(device=DEV).manual_seed(1)
        x = torch.randn(bs, 4, 32, 32, device=DEV, generator=g).to(dtype)
        t = torch.rand(bs, device=DEV, generator=g).to(dtype)
        target = torch.randn(bs, 4, 32, 32, device=DEV, generator=g).float()

        def step(train, fused, seed=None):
            def run():
                os.environ["ZIGMA_FUSED_TRAIN_TAIL"] = "1" if fused else "0"
                m.train(train)
                if seed is not None:
                    torch.manual_seed(seed)
                for p_ in m.parameters():
                    p_.grad = None
                with torch.autocast("cuda", dtype=torch.bfloat16, enabled=amp):
                    out = m.forward_autograd(x, t, None)
                ((out.float() - target) ** 2).mean().backward()
                return out
            return run
        try:
            timing = alternate({"train_fused": step(True, True), "train_per_op": step(True, False), "eval_fused": step(False, True)},
                               reps, 3, warm=2)
            r = {k: v for k, v in timing.items()}
            r["unit"] = "ms per forward + backward"
            r["per_op_over_fused"] = timing["train_per_op"]["median"] / timing["train_fused"]["median"]
            # 3. agreement of the two train-mode paths on one seed, at this size
            outs, grads, rng = {}, {}, {}
            for fused in (True, False):
                o = step(True, fused, seed=1234)()
                outs[fused] = o.detach().float()
                rng[fused] = torch.cuda.get_rng_state()
                grads[fused] = {k: v.grad.float().clone() for k, v in m.named_parameters() if v.grad is not None}
            d = (outs[True] - outs[False]).abs()
            r["same_generator_state"] = bool(torch.equal(rng[True], rng[False]))
            r["out_max_abs_diff"], r["out_max_abs"] = d.max().item(), outs[False].abs().max().item()
            r["grad_worst_rel_l2"] = max(((grads[True][k] - grads[False][k]).norm() / (grads[False][k].norm() + 1e-30)).item()
                                         for k in grads[False])
            res[label] = r
        finally:
            os.environ.pop("ZIGMA_FUSED_TRAIN_TAIL", None)
        del m
        torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("droppath_bench: needs a CUDA device")
    r = {"card": card(), "kernels": kernels(a.reps), "train_step": steps(a.reps)}
    print(json.dumps(r, indent=1))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(r, f, indent=1)


if __name__ == "__main__":
    main()
