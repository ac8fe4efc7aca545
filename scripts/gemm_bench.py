"""wgmma GEMM (zg_gemm_bf16_tn) vs the library GEMM (F.linear) at the eight projection shapes of the hot path: in_proj, out_proj,
x_proj and dt_proj of BASELINE config 2 (D 640, bs 64) and of the D 768 models (FacesHQ, bs 32).

    python scripts/gemm_bench.py [--lib A.so [--lib B.so ...]] [--repeats 7] [--launches 20] [--json OUT]

Each repeat runs every build named by --lib (default: the in-tree build) in a process of its own (ZIGMA_B200_LIB selects it), the builds
alternating, so a slow phase of a shared machine hits all of them alike.  A process times each shape over `launches` back-to-back launches
between CUDA events, for the wgmma kernel and F.linear alike, after a warm-up.  The report gives per shape and build the median and min-max
over the repeats, the card's name, power limit and maximum SM clock, and whether the builds' outputs are bit-identical (seeded inputs)."""
import argparse
import hashlib
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SHAPES = [  # name, M, N, K
    ("in_proj", 65536, 2560, 640), ("out_proj", 65536, 640, 1280), ("x_proj", 65536, 72, 1280), ("dt_proj", 65536, 1280, 40),
    ("in_proj_768", 131072, 3072, 768), ("out_proj_768", 131072, 768, 1536), ("x_proj_768", 131072, 80, 1536), ("dt_proj_768", 131072, 1536, 48),
]


def worker(launches, digest):
    sys.path.insert(0, ROOT)
    import torch
    import torch.nn.functional as F
    from zigma_b200.gemm import linear_bf16

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

    res = {}
    gen = torch.Generator(device="cuda").manual_seed(0)
    for name, M, N, K in SHAPES:
        Kp = (K + 7) // 8 * 8          # x_dbl[:, :R] of dt_proj: a column slice with a padded row pitch, as the engine passes it
        x = torch.randn(M, Kp, device="cuda", generator=gen).bfloat16()[:, :K]
        w = (torch.randn(N, Kp, device="cuda", generator=gen) / K ** 0.5).bfloat16()[:, :K]
        out = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
        ent = {"ours_ms": timeit(lambda: linear_bf16(x, w, out=out)), "lib_ms": timeit(lambda: F.linear(x, w))}
        if digest:
            linear_bf16(x, w, out=out)
            ent["sha1"] = hashlib.sha1(out.view(torch.int16).cpu().numpy().tobytes()).hexdigest()
            ent["max_abs_diff_vs_lib"] = (out.float() - F.linear(x, w).float()).abs().max().item()
        res[name] = ent
        del x, w, out
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
    a = ap.parse_args()
    if a.worker:
        return worker(a.launches, a.digest)
    libs = [os.path.abspath(p) for p in (a.lib or [os.path.join(ROOT, "zigma_b200", "lib", "libzigma_b200.so")])]
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()
    runs = {lib: [] for lib in libs}
    for rep in range(a.repeats):
        for lib in (libs if rep % 2 == 0 else libs[::-1]):
            env = dict(os.environ, ZIGMA_B200_LIB=lib)
            cmd = [sys.executable, os.path.abspath(__file__), "--worker", "--launches", str(a.launches)] + (["--digest"] if rep < 2 else [])
            p = subprocess.run(cmd, env=env, capture_output=True, text=True)
            line = [l for l in p.stdout.splitlines() if l.startswith("RESULT ")]
            if p.returncode != 0 or not line:
                sys.exit(f"worker failed for {lib}:\n{p.stdout[-2000:]}\n{p.stderr[-4000:]}")
            runs[lib].append(json.loads(line[0][7:]))
    stat = lambda v: {"median": statistics.median(v), "min": min(v), "max": max(v)}
    report = {"card": card[0] if card else "unknown", "repeats": a.repeats, "launches": a.launches, "libs": libs, "shapes": {}}
    print(f"card (name, power limit, max SM clock): {report['card']}; medians [min-max] of {a.repeats} alternated repeats x {a.launches} launches, us")
    for name, M, N, K in SHAPES:
        ent = {"M": M, "N": N, "K": K, "builds": {}}
        lib_all = [r[name]["lib_ms"] for lib in libs for r in runs[lib]]
        ent["library"] = stat(lib_all)
        row = f"{name:13s} {M:6d} x {N:4d} x {K:4d}  library {1e3 * ent['library']['median']:7.1f}"
        for i, lib in enumerate(libs):
            s = stat([r[name]["ours_ms"] for r in runs[lib]])
            shas = {r[name]["sha1"] for r in runs[lib] if "sha1" in r[name]}
            ent["builds"][lib] = dict(s, sha1=sorted(shas), max_abs_diff_vs_lib=runs[lib][0][name]["max_abs_diff_vs_lib"])
            row += f"  | [{i}] {1e3 * s['median']:7.1f} [{1e3 * s['min']:6.1f}-{1e3 * s['max']:6.1f}] ({ent['library']['median'] / s['median']:.2f}x lib)"
        ent["bit_identical"] = len({tuple(b["sha1"]) for b in ent["builds"].values()}) == 1 and all(len(b["sha1"]) == 1 for b in ent["builds"].values())
        row += "  same bits" if ent["bit_identical"] else "  BITS DIFFER"
        print(row)
        report["shapes"][name] = ent
    for i, lib in enumerate(libs):
        for tag, names in (("config 2", [s[0] for s in SHAPES[:4]]), ("D 768", [s[0] for s in SHAPES[4:]])):
            ours = sum(report["shapes"][n]["builds"][lib]["median"] for n in names)
            lib_t = sum(report["shapes"][n]["library"]["median"] for n in names)
            print(f"[{i}] {lib}: four projections of {tag}: {1e3 * ours:.1f} us = {ours / lib_t:.2f}x the library's {1e3 * lib_t:.1f} us")
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        json.dump(report, open(a.json, "w"), indent=1)


if __name__ == "__main__":
    main()
