"""Selective-scan forward alone at every scan shape bench.py runs, for one or more builds of the library.

    python scripts/scan_sweep.py [--lib A.so [--lib B.so ...]] [--repeats 7] [--launches 20] [--json OUT]

Shapes (bf16, dstate 16, token-major, z gathered through the zigzag table as the engine passes it): zigzag8_b1 (bs 64 x E 1280 x
L 1024), the second sweep of sweep2_b1 (same shape, reversed accumulating output, no table: the other kernel instantiation),
faceshq1024 (bs 32 x E 1536 x L 4096) and the two layer shapes of ucf101_sst (256 sequences of 256 spatial tokens, 4096 sequences
of 16 frames; E 1536).  Each repeat runs every build named by --lib (default: the in-tree build) in a process of its own
(ZIGMA_B200_LIB selects it, and the process imports the package of the tree the library was built in, <tree>/zigma_b200/lib/),
the builds alternating, so a slow phase of a shared machine hits all of them alike.  A process times
each shape over `launches` back-to-back launches between CUDA events after a warm-up, and reads the launch's grid and block size
from a torch.profiler trace.  The report gives per shape and build the median and min-max over the repeats, the card's name,
power limit and maximum SM clock, and whether the builds' outputs are bit-identical (seeded inputs)."""
import argparse
import hashlib
import json
import os
import statistics
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SHAPES = [  # name, batch, E, L, kind
    ("zigzag8_b1", 64, 1280, 1024, "zigzag"), ("sweep2_b1_rev", 64, 1280, 1024, "sweep"), ("faceshq1024", 32, 1536, 4096, "zigzag"),
    ("ucf_spatial", 256, 1536, 256, "zigzag"), ("ucf_temporal", 4096, 1536, 16, "reverse"),
]


def launch_geometry(fn):
    """(grid, block) of the selective-scan forward kernel `fn` launches, from a torch.profiler trace."""
    import torch
    from torch.profiler import profile, ProfilerActivity
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "trace.json")
        prof.export_chrome_trace(path)
        events = json.load(open(path))["traceEvents"]
    for e in events:
        if e.get("cat") == "kernel" and "scan_fwd" in e.get("name", ""):
            return e["args"].get("grid"), e["args"].get("block")
    return None, None


def worker(tree, launches, digest):
    sys.path.insert(0, tree)
    import torch
    from zigma_b200 import zigzag_path, _lib
    from zigma_b200.selective_scan_interface import _scan_fwd

    def timeit(fn):
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(launches):
            fn()
        b.record()
        torch.cuda.synchronize()
        return a.elapsed_time(b) / launches

    dev, dtype, N = "cuda", torch.bfloat16, 16
    res = {}
    for name, bs, E, L, kind in SHAPES:
        R = E // 32
        gen = torch.Generator(device=dev).manual_seed(0)
        xz = torch.randn(bs, L, 2 * E, device=dev, generator=gen).to(dtype)
        xc = torch.randn(bs, L, E, device=dev, generator=gen).to(dtype)
        dl = (0.5 * torch.rand(bs, L, E, device=dev, generator=gen)).to(dtype)
        xdbl = torch.randn(bs, L, R + 2 * N, device=dev, generator=gen).to(dtype)
        A = -0.5 * torch.rand(E, N, device=dev, generator=gen)
        Dp, bias = torch.randn(E, device=dev, generator=gen), 0.5 * torch.rand(E, device=dev, generator=gen)
        side = int(round(L ** 0.5))
        if kind == "zigzag":
            perm = torch.from_numpy(zigzag_path(side)[1]).to(dev).to(torch.int32)
        elif kind == "reverse":
            perm = torch.arange(L - 1, -1, -1, device=dev, dtype=torch.int32)
        else:
            perm = None
        Bv = xdbl[:, :, R:R + N].permute(0, 2, 1).unsqueeze(1)
        Cv = xdbl[:, :, R + N:].permute(0, 2, 1).unsqueeze(1)
        out = torch.zeros(bs, L, E, device=dev, dtype=dtype).transpose(1, 2)
        extra = dict(out_reverse=True, out_accumulate=True) if kind == "sweep" else {}
        call = lambda: _scan_fwd(xc.transpose(1, 2), dl.transpose(1, 2), A, Bv, Cv, Dp, xz[:, :, E:].transpose(1, 2), bias, True,
                                 z_rowmap=perm, want_last_state=False, out=out, **extra)
        ent = {"ms": timeit(call), "kernel": _lib.last_scan_kernel().split(" ")[0]}
        if digest:
            grid, block = launch_geometry(call)
            ent["grid"], ent["block"] = grid, block
            out.zero_()
            call()      # (the accumulating sweep: one launch onto zeros)
            ent["sha1"] = hashlib.sha1(out.contiguous().view(torch.int16).cpu().numpy().tobytes()).hexdigest()
        res[name] = ent
        del xz, xc, dl, xdbl, out
        torch.cuda.empty_cache()
    print("RESULT " + json.dumps(res))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", action="append", default=None, help="libzigma_b200.so to time (repeatable); default: the in-tree build")
    ap.add_argument("--repeats", type=int, default=7)
    ap.add_argument("--launches", type=int, default=20)
    ap.add_argument("--json", default=None, help="also write the report here")
    ap.add_argument("--worker", action="store_true", help=argparse.SUPPRESS)
    ap.add_argument("--digest", action="store_true", help=argparse.SUPPRESS)
    ap.add_argument("--tree", default=ROOT, help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.worker:
        return worker(a.tree, a.launches, a.digest)
    libs = [os.path.abspath(p) for p in (a.lib or [os.path.join(ROOT, "zigma_b200", "lib", "libzigma_b200.so")])]
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()
    runs = {lib: [] for lib in libs}
    for rep in range(a.repeats):
        for lib in (libs if rep % 2 == 0 else libs[::-1]):
            env = dict(os.environ, ZIGMA_B200_LIB=lib)
            tree = os.path.dirname(os.path.dirname(os.path.dirname(lib)))
            cmd = [sys.executable, os.path.abspath(__file__), "--worker", "--tree", tree, "--launches", str(a.launches)] + (["--digest"] if rep < 2 else [])
            p = subprocess.run(cmd, env=env, capture_output=True, text=True)
            line = [l for l in p.stdout.splitlines() if l.startswith("RESULT ")]
            if p.returncode != 0 or not line:
                sys.exit(f"worker failed for {lib}:\n{p.stdout[-2000:]}\n{p.stderr[-4000:]}")
            runs[lib].append(json.loads(line[0][7:]))
    stat = lambda v: {"median": statistics.median(v), "min": min(v), "max": max(v)}
    report = {"card": card[0] if card else "unknown", "repeats": a.repeats, "launches": a.launches, "libs": libs, "shapes": {}}
    print(f"card (name, power limit, max SM clock): {report['card']}; medians [min-max] of {a.repeats} alternated repeats x {a.launches} launches, ms")
    for name, bs, E, L, kind in SHAPES:
        ent = {"batch": bs, "E": E, "L": L, "builds": {}}
        row = f"{name:14s} {bs:5d} x {E:4d} x {L:5d}"
        for i, lib in enumerate(libs):
            s = stat([r[name]["ms"] for r in runs[lib]])
            first = runs[lib][0][name]
            shas = {r[name]["sha1"] for r in runs[lib] if "sha1" in r[name]}
            ent["builds"][lib] = dict(s, sha1=sorted(shas), kernel=first["kernel"], grid=first.get("grid"), block=first.get("block"))
            row += f"  | [{i}] {s['median']:.4f} [{s['min']:.4f}-{s['max']:.4f}] grid {first.get('grid')} block {first.get('block')}"
        ent["bit_identical"] = len({tuple(b["sha1"]) for b in ent["builds"].values()}) == 1 and all(len(b["sha1"]) == 1 for b in ent["builds"].values())
        row += "  same bits" if ent["bit_identical"] else "  BITS DIFFER"
        print(row)
        report["shapes"][name] = ent
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        json.dump(report, open(a.json, "w"), indent=1)


if __name__ == "__main__":
    main()
