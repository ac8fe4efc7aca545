"""Block tail alone at the layer shape of BASELINE config 2 (bs 64 x 1024 tokens x D 640, bf16, zigzag row table): the plain entry
(zg_block_tail_fwd: reads the previous tail's normed output as x and writes its own normed) against the rebuild entry
(zg_block_tail_fwd_rebuild: rebuilds x from the residual row and the previous tail's rstd, writes no normed).

    python scripts/tail_bench.py [--repeats 7] [--launches 20]

The two entries alternate within one process, `launches` back-to-back launches between CUDA events per sample; reported are the
median and min-max over the repeats, the bytes each entry moves and the rate that makes, the card's name, power limit and maximum SM
clock, and whether the two give the same bits."""
import argparse
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=7)
    ap.add_argument("--launches", type=int, default=20)
    a = ap.parse_args()
    import torch
    from zigma_b200 import zigzag_path
    from zigma_b200.engine import block_tail
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    dev, dt, eps = "cuda", torch.bfloat16, 1e-5
    B, L, D = 64, 1024, 640
    g = torch.Generator(device=dev).manual_seed(0)
    rnd = lambda *s: torch.randn(*s, device=dev, generator=g)
    mods0, mods1 = rnd(B, 3 * D).to(dt), rnd(B, 3 * D).to(dt)
    w0, w1 = (1 + 0.3 * rnd(D)).to(dt), (1 + 0.3 * rnd(D)).to(dt)
    r0, n0, _, rs0 = block_tail(rnd(B, L, D).to(dt), rnd(B, L, D).to(dt), mods0[:, :D], mods0[:, D:2 * D], mods0[:, 2 * D:], w0,
                                4 * rnd(B, L, D), None, eps, want_rstd=True)
    mix = rnd(B, L, D).to(dt)
    perm = torch.from_numpy(zigzag_path(32)[1]).to(dev).to(torch.int32)
    args = (mix, mods1[:, :D], mods1[:, D:2 * D], mods1[:, 2 * D:], w1, r0, perm, eps)
    runs = {"plain": lambda: block_tail(n0, *args, want_rstd=True), "rebuild": lambda: block_tail(None, *args, want_rstd=True, x_from=(rs0, w0))}
    same = all(torch.equal(x, y) for x, y in zip(runs["plain"]()[::2], runs["rebuild"]()[::2]))   # residual_out, modded
    # bytes per call: x (plain only), mix, residual (fp32) read; residual_out (fp32), modded, normed (plain only) written
    row = 2 * D
    nbytes = {"plain": B * L * (row + row + 2 * row + 2 * row + row + row), "rebuild": B * L * (row + 2 * row + 2 * row + row)}
    ts = {k: [] for k in runs}
    for rep in range(a.repeats + 1):
        for k in (list(runs) if rep % 2 == 0 else list(runs)[::-1]):
            fn = runs[k]
            s0, s1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s0.record()
            for _ in range(a.launches):
                fn()
            s1.record()
            torch.cuda.synchronize()
            if rep:         # (the first round warms up)
                ts[k].append(1e3 * s0.elapsed_time(s1) / a.launches)
    print(f"card (name, power limit, max SM clock): {card}; bs {B} x L {L} x D {D} bf16; medians [min-max] of {a.repeats} alternated "
          f"repeats x {a.launches} launches; outputs bit-identical: {same}")
    for k, v in ts.items():
        med = statistics.median(v)
        print(f"{k:8s} {med:7.1f} us [{min(v):6.1f}-{max(v):6.1f}]  {nbytes[k] / 1e6:6.1f} MB -> {nbytes[k] / med / 1e6:5.2f} TB/s")


if __name__ == "__main__":
    main()
