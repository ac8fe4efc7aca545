"""Every instantiation of the hand-written wgmma GEMM (zg_gemm_bf16_tn, zg::gemm_bf16_tn_kernel<BN, CL>) against plain fp64 restatements
of C[M, N] = A[M, K] B[N, K]^T (+ bias[N]), at the engine's shapes and at the edges of the ring, the tiles and the epilogues.

Two references, both computed with fp64 matmuls on the device in row blocks (at most 2^23 elements of C per block):
* exact (primary): A and B hold integers in [-4, 4], the bias integers in [-64, 64], all exact in bf16.  Every partial sum is an
  integer below 2^24 for K <= 8192, so an fp32 accumulator forms it exactly in any order, and C must be the exact product rounded
  once to bf16, to nearest even, bit for bit.  The CPU self-checks below show that the matrix holds elements where rounding toward
  zero differs from nearest-even, ties among them, in both epilogues (TMA store and direct stores).
* fp64 bound (realistic data: N(0,1) activations, weights scaled by 1/sqrt(K), N(0,1) bias): per element, with
  M = sum_k |a_mk b_nk| + |bias_n|, |a - e| <= max(1 ulp_bf16(e), C_GEMM ceil(K/16) 2^-24 M + 1 ulp), one rounding (perhaps a
  truncation) per k16 wgmma step.  The CPU self-checks show that it accepts a sequential fp32 sum and rejects a kernel that drops
  one k-block, the bias, or shifts one column group.  No mismatch fraction is asserted on this data: the exact suite pins the
  rounding.

The matrix is a covering design: each instantiation, forced through ZG_GEMM_BN / ZG_GEMM_CLUSTER (read on every call), takes every
value of every axis it can: M (one tile row, two, three -- an idle CTA in the last cluster of 2 --, six -- two idle in the last
cluster of 4 --, and enough tile rows that every resident cluster runs several tiles, carrying ring stage and phase from tile to
tile), N (one tile, ragged inside the last 64-column TMA chunk or the 16- / 32-column direct tail, one valid column or one valid
8-column group in the last tile -- the other TMA chunks empty --, fewer than 8 columns), K (the patch embedding's 8 and 16, dt_proj's 40, around the ring depth S: 64 (S - 1), 64 S + 8,
64 (2 S + 1) - 24, and 1280), the padding of A and B (NaN beyond K), the bias, and the epilogue (TMA store; direct stores forced
by ldc % 8 != 0, by a C base that is not 16-byte aligned, or by a row scatter).  C is always a window into a sentinel-filled
buffer that must keep the sentinel outside [M, N].  The engine's GEMM shapes run at full size with the automatic choice.

The achieved worst ulp, fraction of the bound and accumulation constant of every check go to $ZIGMA_PARITY_LOG when it names a file.
The last part is the inventory: the library holds exactly the 14 instantiations of INSTANCES, the case table reaches all of them
through zg_gemm_kernel_choice, and on the GPU each case launches the kernel the choice function predicts."""
import math
import os
import re
import shutil
import subprocess
from collections import namedtuple

import numpy as np
import pytest
import torch

from util import _log, check_close, check_elem, ulp

DEV = "cuda"
gpu = pytest.mark.gpu
F64, BF16 = torch.float64, torch.bfloat16

# fp32 accumulation constant of the fp64 bound: the worst (|a - e| - half an ulp of the output) / (ceil(K/16) 2^-24 M) measured on
# an H100 80GB HBM3 (700 W) over the whole file, 0.93 (at K = 16, one k16 step), times 4, rounded up.
C_GEMM = 4

WIDTHS = (64, 80, 128, 160, 256)
# a CTA multicasts BN / CL rows of the weight tile, which must be whole 8-row swizzle groups: no <80, 4>
INSTANCES = sorted((bn, cl) for bn in WIDTHS for cl in (1, 2, 4) if (bn // cl) % 8 == 0)
SENTINEL = -0x3e01                        # int16 view of the bf16 that fills C's buffer outside the window (bits 0xC1FF, -31.875)
ROW_BLOCK = 1 << 23                       # elements of C per fp64 reference block (about 1 GB of fp64 temporaries)


def stages(bn):
    """Ring depth of gemm_stages (gemm_wgmma.cu): (128 + BN) x 64 bf16 stages next to the epilogue staging, at most 8."""
    avail = 227 * 1024 - 8 * 2 * 16 * 128 - 2048
    return min(8, avail // ((128 + bn) * 64 * 2))


def predicted(M, N, bn=None, cl=None):
    """(BN, CL) for an M x N call: the rule of gemm_choice (gemm_wgmma.cu) restated, with the forced width / cluster of a case."""
    if bn is None:
        def waste(b):
            padded = -(-N // b) * b
            return (padded - N) / padded
        fits = [b for b in (256, 160, 128, 80, 64) if waste(b) <= 0.05]
        bn = fits[0] if fits else _least_waste(waste)
    cl = 2 if cl is None else cl
    while cl > 1 and (-(-M // 128) < cl or (bn // cl) % 8):
        cl //= 2
    return bn, cl


def _least_waste(waste):
    best = 64                               # (the C loop: start at 64, take a candidate only if it wastes strictly less)
    for b in (256, 160, 128, 80, 64):
        if waste(b) < waste(best) - 1e-9:
            best = b
    return best


# ------------------------------------------------------------------------------------------------ the case table
Case = namedtuple("Case", "id M N K bn cl layout bias pad kernel")
M_MANY = 400 * 128 - 37                 # 400 tile rows: every resident cluster (132 SMs) runs at least 3 tiles, even with one tile column
M_VALUES = (1, 129, 3 * 128, 5 * 128 + 7, M_MANY)
M_LAYOUT, RPB = 6 * 128 - 10, 379        # the layout cases: 6 tile rows (two idle CTAs in the last cluster of 4); scatter in 2 batches
LAYOUTS = ("tma", "ldc_odd", "c_unaligned", "scatter")


def _matrix():
    cases = []
    for bn, cl in INSTANCES:
        S = stages(bn)
        ms = [m for m in M_VALUES if -(-m // 128) >= cl]
        ns = (bn, 3 * bn - 8, 2 * bn + 1, 2 * bn + 8, 7)
        ks = (8, 16, 40, 64 * (S - 1), 64 * S + 8, 64 * (2 * S + 1) - 24, 1280)
        for i in range(7):                  # covering: every M, N and K value of this instantiation at least once
            M, N, K = ms[i % len(ms)], ns[i % len(ns)], ks[i]
            cases.append(Case(f"bn{bn}_cl{cl}_m{M}_n{N}_k{K}_{'b' if i % 2 == 0 else 'nb'}_p{8 * (i % 3 == 1)}",
                              M, N, K, bn, cl, "tma", i % 2 == 0, 8 * (i % 3 == 1), predicted(M, N, bn, cl)))
        N, K = 3 * bn - 8, 64 * S + 8       # one ragged shape per instantiation in every other epilogue
        for j, layout in enumerate(LAYOUTS[1:]):
            cases.append(Case(f"bn{bn}_cl{cl}_{layout}", M_LAYOUT, N, K, bn, cl, layout, j != 1, 8 * (j == 0),
                              predicted(M_LAYOUT, N, bn, cl)))
    return cases


MATRIX = _matrix()

# the engine's GEMMs at full size, automatic choice: (name, M, N, K, bias, kernel it must get)
ENGINE = [
    ("in_proj", 65536, 2560, 640, False, (256, 2)),            # BASELINE config 2 (D 640, bs 64, 32 x 32 latents, patch 1)
    ("out_proj", 65536, 640, 1280, False, (160, 2)),
    ("x_proj", 65536, 72, 1280, False, (80, 2)),
    ("dt_proj", 65536, 1280, 40, False, (256, 2)),
    ("in_proj_d768", 131072, 3072, 768, False, (256, 2)),      # the D 768 models
    ("out_proj_d768", 131072, 768, 1536, False, (256, 2)),
    ("x_proj_d768", 131072, 80, 1536, False, (80, 2)),
    ("dt_proj_d768", 131072, 1536, 48, False, (256, 2)),
    ("adaln", 64, 34560, 640, True, (256, 1)),                 # every block's adaLN Linear in one GEMM: depth 18 x 3 x D, one tile row
    ("patch_embed", 65536, 640, 8, True, (160, 2)),
    ("patch_embed_d768", 131072, 768, 16, True, (256, 2)),
    ("unembed", 65536, 4, 640, True, (64, 2)),                 # N = patch^2 x output channels, K = D
    ("unembed_d768", 131072, 16, 768, True, (64, 2)),
]


# ------------------------------------------------------------------------------------------------ operands and layouts
def _ints(gen, shape, lo, hi):
    return torch.randint(lo, hi + 1, shape, generator=gen, dtype=torch.int8, device=gen.device)


def operands(M, N, K, bias, exact, seed, device):
    """(a, w, b) as bf16 on `device`: integers for the exact reference, realistic data for the fp64 bound.  Drawn on the CPU for the
    matrix (so that the CPU self-checks see the same data), on the device for the engine shapes."""
    gen = torch.Generator(device=device).manual_seed(seed)
    if exact:
        a, w = _ints(gen, (M, K), -4, 4), _ints(gen, (N, K), -4, 4)
        b = _ints(gen, (N,), -64, 64) if bias else None
    else:
        a = torch.randn(M, K, generator=gen, device=device)
        w = torch.randn(N, K, generator=gen, device=device) / math.sqrt(K)
        b = torch.randn(N, generator=gen, device=device) if bias else None
    return a.to(BF16), w.to(BF16), None if b is None else b.to(BF16)


def case_operands(case, exact):
    seed = sum((i + 1) * ord(c) for i, c in enumerate(case.id))       # (stable across processes, unlike hash())
    return operands(case.M, case.N, case.K, case.bias, exact, seed=seed, device="cpu")


def padded(t, pad, device):
    """t (rows, K) as a column window of a NaN-filled (rows, round8(K) + pad) buffer on `device`."""
    rows, K = t.shape
    buf = torch.full((rows, -(-K // 8) * 8 + pad), float("nan"), dtype=BF16, device=device)
    buf[:, :K] = t.to(device)
    return buf[:, :K]


def row_map(M, rpb, device, seed=0):
    """(out_rowmap, dest): a random permutation of the rows of each batch of rpb rows; dest[m] is the row of C that row m of the
    product lands in."""
    gen = torch.Generator().manual_seed(seed)
    perm = torch.randperm(rpb, generator=gen).to(torch.int32)
    dest = (torch.arange(M) // rpb) * rpb + perm.long()[torch.arange(M) % rpb]
    return perm.to(device), dest.to(device)


class Window:
    """C as an [M, N] window (row stride ldc) into a sentinel-filled bf16 buffer, for one epilogue layout."""

    def __init__(self, M, N, layout, device=DEV):
        self.ldc = -(-N // 8) * 8 + 8 + (3 if layout == "ldc_odd" else 0)
        self.off = 8 * self.ldc + (1 if layout == "c_unaligned" else 0)    # 8 sentinel rows in front; +1 element: 2-byte aligned base
        self.buf = torch.full((self.off + (M + 2) * self.ldc + 8,), 0, dtype=torch.int16, device=device).fill_(SENTINEL).view(BF16)
        self.out = self.buf.as_strided((M, N), (self.ldc, 1), self.off)
        self.M, self.N = M, N

    def untouched(self):
        """Number of buffer elements outside the window that lost the sentinel."""
        inside = torch.zeros(self.buf.numel(), dtype=torch.bool, device=self.buf.device)
        inside.as_strided((self.M, self.N), (self.ldc, 1), self.off).fill_(True)
        return int(((self.buf.view(torch.int16) != SENTINEL) & ~inside).sum())


def run(case, a, w, b, monkeypatch, device=DEV):
    """The kernel on one case: forced width / cluster, padded operands, C window of the case's layout.  Returns (C in product row
    order, window)."""
    if case.bn is None:
        monkeypatch.delenv("ZG_GEMM_BN", raising=False)
        monkeypatch.delenv("ZG_GEMM_CLUSTER", raising=False)
    else:
        monkeypatch.setenv("ZG_GEMM_BN", str(case.bn))
        monkeypatch.setenv("ZG_GEMM_CLUSTER", str(case.cl))
    from zigma_b200.gemm import linear_bf16
    win = Window(case.M, case.N, case.layout, device)
    A, W = padded(a, case.pad, device), padded(w, case.pad, device)
    bias = None if b is None else b.to(device)
    if case.layout == "scatter":
        rowmap, dest = row_map(case.M, RPB, device)
        linear_bf16(A, W, bias, out=win.out, out_rowmap=rowmap, rows_per_batch=RPB)
        return win.out[dest], win
    linear_bf16(A, W, bias, out=win.out)
    return win.out, win


# ------------------------------------------------------------------------------------------------ fp64 references
def _blocks(M, N):
    step = max(1, min(8192, ROW_BLOCK // N))
    return [(r, min(M, r + step)) for r in range(0, M, step)]


def exact_product(a, w, b):
    """fp64 a w^T + b.  On integer-valued operands every sum is an integer below 2^53, so it is exact, and .to(bf16) rounds it once
    to nearest even (through fp32, which holds every integer below 2^24 exactly)."""
    e = a.double() @ w.double().t()
    return e if b is None else e + b.double()


def check_exact(what, got, a, w, b):
    """got == the exactly rounded product bit for bit, in row blocks; logs how many elements needed rounding and how many of them
    were ties."""
    bad, rounded, ties, first = 0, 0, 0, None
    for r0, r1 in _blocks(*got.shape):
        e = exact_product(a[r0:r1], w, b)
        diff = got[r0:r1].view(torch.int16) != e.to(BF16).view(torch.int16)
        n = int(diff.sum())
        if n and first is None:
            idx = diff.nonzero()[:4]
            first = [(r0 + int(i), int(j), got[r0 + int(i), int(j)].item(), e[i, j].item()) for i, j in idx.tolist()]
            mags = e[diff].abs()
            first.append(f"|exact| of the mismatches in [{mags.min().item():g}, {mags.max().item():g}]")
        bad += n
        r, t = rounding_counts(e)
        rounded, ties = rounded + r, ties + t
    _log(what, BF16, exact_mismatches=bad, rounded=rounded, ties=ties, numel=got.numel())
    assert bad == 0, f"{what}: {bad}/{got.numel()} elements differ from the exactly rounded product; first (row, col, got, exact): {first}"


def rounding_counts(e):
    """(elements whose exact integer value is not a bf16, of which exact ties) among the fp64 values e."""
    s = ulp(e, BF16)
    frac = e.abs() / s - torch.floor(e.abs() / s)
    return int((frac != 0).sum()), int((frac == 0.5).sum())


def check_bound(what, got, a, w, b, c=C_GEMM):
    """The fp64 bound, in row blocks (check_elem per block); logs the worst ulp and the observed accumulation constant."""
    K = a.shape[1]
    steps = -(-K // 16)
    wd = w.double()
    wa = wd.abs()
    worst_ulp, worst_c = 0.0, 0.0
    for r0, r1 in _blocks(*got.shape):
        ad = a[r0:r1].double()
        e = ad @ wd.t()
        Mg = ad.abs() @ wa.t()
        if b is not None:
            e, Mg = e + b.double(), Mg + b.double().abs()
        g = got[r0:r1].double()
        diff = (g - e).abs()
        half = 0.5 * torch.maximum(ulp(e, BF16), ulp(g, BF16))
        worst_c = max(worst_c, ((diff - half).clamp(min=0) / (steps * 2.0 ** -24 * Mg.clamp(min=1e-300))).max().item())
        worst_ulp = max(worst_ulp, (diff / ulp(e, BF16)).max().item())
        check_elem(f"{what} rows {r0}:{r1}", got[r0:r1], e, Mg, max_ulp=1, c_f32=c * steps, mismatch=1.0)
    _log(what, BF16, worst_ulp=worst_ulp, worst_c_accum=worst_c, K=K, numel=got.numel())
    return worst_c


# ------------------------------------------------------------------------------------------------ GPU: the matrix
@gpu
@pytest.mark.parametrize("case", MATRIX, ids=[c.id for c in MATRIX])
def test_matrix_exact(case, monkeypatch):
    a, w, b = case_operands(case, exact=True)
    got, win = run(case, a, w, b, monkeypatch)
    a, w = a.to(DEV), w.to(DEV)
    check_exact(f"gemm<{case.kernel[0]},{case.kernel[1]}> {case.id} exact", got, a, w, None if b is None else b.to(DEV))
    assert win.untouched() == 0, f"{case.id}: the kernel wrote outside the [M, N] window of C"


@gpu
@pytest.mark.parametrize("case", MATRIX, ids=[c.id for c in MATRIX])
def test_matrix_fp64_bound(case, monkeypatch):
    a, w, b = case_operands(case, exact=False)
    got, win = run(case, a, w, b, monkeypatch)
    check_bound(f"gemm<{case.kernel[0]},{case.kernel[1]}> {case.id} fp64", got, a.to(DEV), w.to(DEV), None if b is None else b.to(DEV))
    assert win.untouched() == 0, f"{case.id}: the kernel wrote outside the [M, N] window of C"


@gpu
@pytest.mark.parametrize("name,M,N,K,bias,kernel", ENGINE, ids=[e[0] for e in ENGINE])
def test_engine_shapes(name, M, N, K, bias, kernel, monkeypatch):
    """The engine's GEMMs at full size with the automatic choice, against both references."""
    case = Case(name, M, N, K, None, None, "tma", bias, 0, kernel)
    assert predicted(M, N) == kernel
    for exact in (True, False):
        a, w, b = operands(M, N, K, bias, exact, seed=M + N + K, device=DEV)
        got, win = run(case, a, w, b, monkeypatch)
        if exact:
            check_exact(f"gemm<{kernel[0]},{kernel[1]}> {name} exact", got, a, w, b)
        else:
            check_bound(f"gemm<{kernel[0]},{kernel[1]}> {name} fp64", got, a, w, b)
        assert win.untouched() == 0
        del got, win, a, w, b
    torch.cuda.empty_cache()


SHAPES = [
    # M, N, K                      what
    (4096, 2560, 640),            # in_proj  (bs=4 slice of BASELINE config 2)
    (4096, 640, 1280),            # out_proj
    (4096, 72, 1280),             # x_proj   (N not a tile multiple)
    (4096, 1280, 40),             # dt_proj  (K < one k-block: TMA zero fill)
    (1000, 200, 136),             # everything ragged
    (128, 64, 64), (1, 8, 8), (129, 257, 72),
    (4096, 80, 1536), (4096, 768, 1536),   # x_proj / out_proj of the D = 768 models (80-wide tile; 3 x 256)
    (300, 5184, 72),              # 256-wide tiles whose last column tile holds 64 valid columns: its other chunks store nothing
    (300, 160, 64), (257, 150, 200), (520, 330, 96),   # 160-wide tiles: exact, ragged in N (tail columns by direct stores), two tiles + ragged
]
SHAPE_CASES = [Case(f"{M}x{N}x{K}_{'b' if bias else 'nb'}", M, N, K, None, None, "tma", bias, 8, predicted(M, N))
               for M, N, K in SHAPES for bias in (False, True)]


@gpu
@pytest.mark.parametrize("M,N,K", SHAPES)
@pytest.mark.parametrize("has_bias", [False, True])
def test_gemm_shapes(M, N, K, has_bias, monkeypatch):
    """Projection-sized and ragged shapes with the automatic choice, A and B with a padded pitch, against both references."""
    case = Case(f"{M}x{N}x{K}", M, N, K, None, None, "tma", has_bias, 8, predicted(M, N))
    for exact in (True, False):
        a, w, b = operands(M, N, K, has_bias, exact, seed=M + N + K, device=DEV)
        got, win = run(case, a, w, b, monkeypatch)
        what = f"gemm<{case.kernel[0]},{case.kernel[1]}> {M}x{N}x{K} bias={has_bias}"
        if exact:
            check_exact(what + " exact", got, a, w, b)
        else:
            check_bound(what + " fp64", got, a, w, b)
        assert win.untouched() == 0


@gpu
def test_gemm_row_scatter_and_views():
    """out_rowmap scatters each batch's rows (out_proj + backward_permutation fused); A given as a
    column slice of a wider matrix (dt_proj reads x_dbl[:, :R] in place)."""
    from zigma_b200.gemm import linear_bf16
    import zigma_b200
    B, L, K, N = 3, 64, 72, 96
    x_dbl = torch.randn(B * L, K, device=DEV).bfloat16()
    w = torch.randn(N, 40, device=DEV).bfloat16()
    rev = torch.from_numpy(zigma_b200.reverse_permut_np(zigma_b200.zigzag_path(8)[2])).to(DEV)
    out = linear_bf16(x_dbl[:, :40], w, out_rowmap=rev.to(torch.int32), rows_per_batch=L)
    ref = (x_dbl[:, :40].float() @ w.float().t()).view(B, L, N)
    want = torch.empty_like(ref)
    want[:, rev] = ref                                   # row m lands at row rev[m]
    check_close(out.view(B, L, N), want, "gemm row scatter", rtol=8e-3, atol=1e-5, max_strict_viol=1.0)
    # the out_proj shape of the D = 640 models with the scatter (160-wide tiles, direct-store epilogue for every column)
    y = torch.randn(B * L, 128, device=DEV).bfloat16()
    w2 = (torch.randn(640, 128, device=DEV) / 128 ** 0.5).bfloat16()
    out2 = linear_bf16(y, w2, out_rowmap=rev.to(torch.int32), rows_per_batch=L)
    ref2 = (y.float() @ w2.float().t()).view(B, L, 640)
    want2 = torch.empty_like(ref2)
    want2[:, rev] = ref2
    check_close(out2.view(B, L, 640), want2, "gemm row scatter N=640", rtol=8e-3, atol=1e-5, max_strict_viol=1.0)


@gpu
def test_engine_with_tcgen05_gemms(monkeypatch):
    """Whole bf16 model with the projections routed through zg_gemm_bf16_tn (ZIGMA_TCGEN05=1, the historical name of the switch) == library-GEMM engine."""
    from oracle import synth
    from oracle.gen_golden import model_io
    from util import model_case
    from zigma_b200 import ZigMa
    g, cfg, shapes = model_case("tiny_zigzag8_bf16")
    outs = {}
    for flag in ("0", "1"):
        monkeypatch.setenv("ZIGMA_TCGEN05", flag)
        m = ZigMa(device=DEV, dtype=torch.bfloat16, **cfg).eval()
        m.load_state_dict(synth.synth_state_dict(shapes, seed=0, dtype=torch.bfloat16))
        x, tt, _ = model_io(cfg, 2)
        with torch.no_grad():
            outs[flag] = m(x.to(DEV).bfloat16(), tt.to(DEV).bfloat16()).float()
    check_close(outs["1"], outs["0"], "engine wgmma vs library GEMMs", rtol=3e-2, atol=3e-2, scale_atol=False, max_strict_viol=1.0)
    check_close(outs["1"], g["out"], "engine wgmma vs reference bf16", rtol=5e-2, atol=5e-2, scale_atol=False, max_strict_viol=1.0)


# ------------------------------------------------------------------------------------------------ GPU: invariants (random data, bit equality)
@gpu
@pytest.mark.parametrize("bn", WIDTHS)
def test_invariants(bn, monkeypatch):
    """Per tile width, on random data: every cluster size gives the same C (each tile sums its k-blocks in the same order), the
    direct-store epilogues give the TMA store's C, the row scatter is the unscattered C permuted, and a repeated call repeats C."""
    from zigma_b200.gemm import linear_bf16
    M, N, K = 2000, 3 * bn - 8, 1280
    a, w, b = operands(M, N, K, True, exact=False, seed=bn, device=DEV)
    monkeypatch.setenv("ZG_GEMM_BN", str(bn))
    outs = {}
    for cl in sorted({cl for b_, cl in INSTANCES if b_ == bn}):
        monkeypatch.setenv("ZG_GEMM_CLUSTER", str(cl))
        outs[cl] = linear_bf16(a, w, b)
    ref = outs[1].view(torch.int16)
    for cl, o in outs.items():
        assert torch.equal(o.view(torch.int16), ref), f"BN {bn}: clusters of {cl} differ from clusters of 1"
    monkeypatch.setenv("ZG_GEMM_CLUSTER", str(max(outs)))
    for layout in ("ldc_odd", "c_unaligned"):
        win = Window(M, N, layout)
        linear_bf16(a, w, b, out=win.out)
        assert torch.equal(win.out.view(torch.int16), ref), f"BN {bn}: direct stores ({layout}) differ from the TMA store"
        assert win.untouched() == 0
    rowmap, dest = row_map(M, 250, DEV, seed=bn)
    sc = linear_bf16(a, w, b, out_rowmap=rowmap, rows_per_batch=250)
    assert torch.equal(sc[dest].view(torch.int16), ref), f"BN {bn}: row scatter is not the unscattered C permuted"
    again = linear_bf16(a, w, b)
    assert torch.equal(again.view(torch.int16), ref), f"BN {bn}: a repeated call changed C"


# ------------------------------------------------------------------------------------------------ GPU: argument checks of linear_bf16
def _bad_calls():
    """(name, kwargs builder): each call is wrong in one argument, and built so that WITHOUT the check the kernel would still read
    and write only allocated memory at in-range indices (views into larger buffers, in-range row indices)."""
    M, N, K = 300, 96, 64

    def base():
        a = torch.randn(M, K, device=DEV).bfloat16()
        w = torch.randn(N, K, device=DEV).bfloat16()
        return a, w

    def out_short_rows():
        big = torch.zeros(M, N, device=DEV, dtype=BF16)
        return dict(out=big[:M - 1])
    def out_col_stride():
        big = torch.zeros(M, 2 * N, device=DEV, dtype=BF16)
        return dict(out=big[:, ::2])
    def out_fp32():
        return dict(out=torch.zeros(M, N, device=DEV))
    def bias_fp32():
        return dict(bias=torch.randn(N, device=DEV))
    def bias_short():
        return dict(bias=torch.randn(N, device=DEV).bfloat16()[:N - 1])
    def bias_strided():
        return dict(bias=torch.randn(2 * N, device=DEV).bfloat16()[::2])
    def rowmap_int64():
        return dict(out_rowmap=torch.randperm(100, device=DEV), rows_per_batch=100)
    def rowmap_strided():
        big = torch.arange(100, device=DEV, dtype=torch.int32).repeat_interleave(2)   # (the first 100 elements are in range too)
        return dict(out_rowmap=big[::2], rows_per_batch=100)
    def rowmap_short():
        big = torch.arange(100, device=DEV, dtype=torch.int32)
        return dict(out_rowmap=big[:99], rows_per_batch=100)
    calls = [out_short_rows, out_col_stride, out_fp32, bias_fp32, bias_short, bias_strided, rowmap_int64, rowmap_strided, rowmap_short]
    return base, calls


@gpu
@pytest.mark.parametrize("bad", _bad_calls()[1], ids=[f.__name__ for f in _bad_calls()[1]])
def test_linear_bf16_rejects_bad_arguments(bad):
    from zigma_b200.gemm import linear_bf16
    base = _bad_calls()[0]
    a, w = base()
    with pytest.raises(RuntimeError):
        linear_bf16(a, w, **bad())
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------ inventory
GEMM_RE = re.compile(r"zg::gemm_bf16_tn_kernel<\s*(?:\(int\))?(\d+)\s*,\s*(?:\(int\))?(\d+)\s*>")
ENGINE_CASES = [Case(n, M, N, K, None, None, "tma", bias, 0, kern) for n, M, N, K, bias, kern in ENGINE] + SHAPE_CASES


def _tool(name):
    p = os.path.join("/usr/local/cuda/bin", name)
    return shutil.which(name) or (p if os.path.exists(p) else None)


def test_inventory_matches_library():
    """CPU: the zg::gemm_bf16_tn_kernel instantiations in the built library are exactly INSTANCES (14)."""
    assert len(INSTANCES) == 14 and (80, 4) not in INSTANCES
    cuobjdump, filt = _tool("cuobjdump"), _tool("cu++filt")
    if cuobjdump is None or filt is None:
        pytest.skip("cuobjdump / cu++filt not available")
    import __graft_entry__
    __graft_entry__.build()
    from zigma_b200 import _lib
    listing = subprocess.run([cuobjdump, "-elf", _lib.LIB_PATH], check=True, capture_output=True, text=True).stdout
    names = sorted(set(re.findall(r"\.text\.(_Z\S+)", listing)))
    demangled = subprocess.run([filt], input="\n".join(names), check=True, capture_output=True, text=True).stdout.splitlines()
    found = {(int(m.group(1)), int(m.group(2))) for m in map(GEMM_RE.search, demangled) if m}
    assert found == set(INSTANCES), f"in the library: {sorted(found)}"


def test_choice_function_reaches_every_instance(monkeypatch):
    """CPU: zg_gemm_kernel_choice, with each case's settings in the environment, names the kernel the case table records (the rule
    restated in predicted()), and the table reaches all 14 instantiations, half of them from more than one case."""
    from zigma_b200 import _lib
    import __graft_entry__
    __graft_entry__.build()
    seen = {}
    for case in MATRIX + ENGINE_CASES:
        _set_env(case, monkeypatch)
        got = _lib.gemm_kernel_choice(case.M, case.N)
        assert got == case.kernel, f"{case.id}: zg_gemm_kernel_choice says {got}, the table {case.kernel}"
        seen[got] = seen.get(got, 0) + 1
    assert set(seen) == set(INSTANCES), sorted(seen)
    # the forced settings are read per call, and the cluster still halves: too few tile rows, or 80-wide tiles
    monkeypatch.setenv("ZG_GEMM_BN", "80")
    monkeypatch.setenv("ZG_GEMM_CLUSTER", "4")
    assert _lib.gemm_kernel_choice(4096, 72) == (80, 2)
    monkeypatch.setenv("ZG_GEMM_BN", "128")
    assert _lib.gemm_kernel_choice(4096, 72) == (128, 4) and _lib.gemm_kernel_choice(384, 72) == (128, 2)
    assert _lib.gemm_kernel_choice(129, 72) == (128, 2) and _lib.gemm_kernel_choice(128, 72) == (128, 1)
    monkeypatch.setenv("ZG_GEMM_CLUSTER", "3")            # not a cluster size: the default
    monkeypatch.setenv("ZG_GEMM_BN", "96")                # not a width: the automatic rule
    assert _lib.gemm_kernel_choice(4096, 640) == (160, 2)
    with pytest.raises(RuntimeError):
        _lib.gemm_kernel_choice(0, 64)


def test_choice_rule_over_widths(monkeypatch):
    """CPU: the automatic width rule of zg_gemm_kernel_choice equals predicted() for every N up to 4096."""
    from zigma_b200 import _lib
    import __graft_entry__
    __graft_entry__.build()
    monkeypatch.delenv("ZG_GEMM_BN", raising=False)
    monkeypatch.delenv("ZG_GEMM_CLUSTER", raising=False)
    for N in range(1, 4097):
        assert _lib.gemm_kernel_choice(4096, N) == predicted(4096, N), N


def _set_env(case, monkeypatch):
    if case.bn is None:
        monkeypatch.delenv("ZG_GEMM_BN", raising=False)
        monkeypatch.delenv("ZG_GEMM_CLUSTER", raising=False)
    else:
        monkeypatch.setenv("ZG_GEMM_BN", str(case.bn))
        monkeypatch.setenv("ZG_GEMM_CLUSTER", str(case.cl))


@gpu
def test_matrix_launches_predicted_kernels(monkeypatch):
    """The matrix and the engine shapes, run once more on zero operands, one torch.profiler session per case: each case launches
    exactly one kernel (the library's launch counter), every GEMM launch the profiler records is the kernel the case table predicts
    for that case, and together they are exactly INSTANCES.  (The profiler can lose a kernel record now and then, so a case without
    a record only goes unchecked by it; the counter still proves that it launched.)"""
    from torch.profiler import ProfilerActivity, profile
    from zigma_b200 import _lib
    from zigma_b200.gemm import linear_bf16
    cases = MATRIX + ENGINE_CASES
    seen, wrong, unrecorded = set(), [], []
    for case in cases:
        _set_env(case, monkeypatch)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            a = torch.zeros(case.M, -(-case.K // 8) * 8 + case.pad, device=DEV, dtype=BF16)[:, :case.K]
            w = torch.zeros(case.N, -(-case.K // 8) * 8 + case.pad, device=DEV, dtype=BF16)[:, :case.K]
            b = torch.zeros(case.N, device=DEV, dtype=BF16) if case.bias else None
            win = Window(case.M, case.N, case.layout)
            before = _lib.launch_count()
            if case.layout == "scatter":
                rowmap, _ = row_map(case.M, RPB, DEV)
                linear_bf16(a, w, b, out=win.out, out_rowmap=rowmap, rows_per_batch=RPB)
            else:
                linear_bf16(a, w, b, out=win.out)
            assert _lib.launch_count() - before == 1, f"{case.id}: {_lib.launch_count() - before} launches"
            torch.cuda.synchronize()
        got = [(int(m.group(1)), int(m.group(2))) for e in prof.events() for m in [GEMM_RE.search(e.name)] if m]
        assert len(got) <= 1, f"{case.id}: the profiler recorded {got}"
        if not got:
            unrecorded.append(case.id)
        elif got[0] != case.kernel:
            wrong.append((case.id, case.kernel, got[0]))
        seen.update(got)
        del a, w, b, win
    print(f"    {len(cases) - len(unrecorded)}/{len(cases)} launches recorded by the profiler; unrecorded: {unrecorded}")
    assert not wrong, f"cases that launched another kernel than predicted (case, predicted, launched): {wrong[:5]}"
    assert seen == set(INSTANCES), f"recorded: {sorted(seen)}"


# ------------------------------------------------------------------------------------------------ CPU self-checks of the references
def _rne_bf16_int(v):
    """Python integer v (|v| < 2^24) rounded to bf16 (8 significant bits), to nearest, ties to even."""
    m = abs(v)
    if m < 256:
        return v
    shift = m.bit_length() - 8
    q, r = divmod(m, 1 << shift)
    half = 1 << (shift - 1)
    if r > half or (r == half and q % 2):
        q += 1
    return (q << shift) * (1 if v >= 0 else -1)


def test_exact_product_is_integer_arithmetic():
    """CPU: the exactly rounded product == Python integers summed and rounded to nearest even, at K = 1280 and at K = 8192 with the
    largest sums the data allows (|a b| = 16 everywhere: up to 2^17)."""
    for M, N, K in ((6, 5, 1280), (3, 4, 8192)):
        a, w, b = operands(M, N, K, True, True, seed=K, device="cpu")
        if K == 8192:                                       # the largest sums the premise allows: |a b| = 16 everywhere
            a, w = (torch.where(a >= 0, 4, -4).to(BF16), torch.full_like(w, 4))
        got = exact_product(a, w, b).to(BF16).double()
        ai, wi, bi = a.to(torch.int64).tolist(), w.to(torch.int64).tolist(), b.to(torch.int64).tolist()
        for m in range(M):
            for n in range(N):
                v = sum(x * y for x, y in zip(ai[m], wi[n])) + bi[n]
                assert abs(v) < 1 << 24 and got[m, n].item() == _rne_bf16_int(v), (M, N, K, m, n, v, got[m, n].item())


def test_matrix_exercises_rounding():
    """CPU: the integer data of the matrix's cases (all but the many-tile M) holds elements where rounding toward zero and to
    nearest even differ, and exact ties, both in cases that leave through the TMA store and in cases that leave by direct stores."""
    counts = {"tma": [0, 0], "direct": [0, 0]}
    for case in MATRIX:
        if case.M == M_MANY or case.K < 256:
            continue
        a, w, b = case_operands(case, exact=True)
        e = a.double() @ w.double().t() + (0 if b is None else b.double())
        rne = e.to(BF16).double()
        rtz = torch.sign(e) * torch.floor(e.abs() / ulp(e, BF16)) * ulp(e, BF16)
        _, ties = rounding_counts(e)
        kind = "tma" if case.layout == "tma" else "direct"
        counts[kind][0] += int((rne != rtz).sum())
        counts[kind][1] += ties
    for kind, (differ, ties) in counts.items():
        assert differ > 100 and ties > 10, (kind, differ, ties)


def _seq_fp32(a, w, b):
    """Sequential fp32 sum over k, rounded to nearest after every add (numpy), + bias, rounded to bf16."""
    A, W = a.float().numpy(), w.float().numpy()
    acc = np.zeros((A.shape[0], W.shape[0]), dtype=np.float32)
    for k in range(A.shape[1]):
        acc = (acc + np.outer(A[:, k], W[:, k]).astype(np.float32)).astype(np.float32)
    if b is not None:
        acc = (acc + b.float().numpy()[None]).astype(np.float32)
    return torch.from_numpy(acc).to(BF16)


def _ref64(a, w, b):
    e = a.double() @ w.double().t() + (0 if b is None else b.double())
    Mg = a.double().abs() @ w.double().abs().t() + (0 if b is None else b.double().abs())
    return e, Mg


def test_bound_accepts_sequential_fp32_and_rejects_defects():
    """CPU: the fp64 bound accepts a sequential fp32 round-to-nearest sum at the largest K of the file, and rejects one k-block
    dropped, the bias omitted, and one 8-column group shifted by 8 columns."""
    M, N, K = 32, 48, 1536
    a, w, b = operands(M, N, K, True, exact=False, seed=7, device="cpu")
    check_bound("self-check sequential fp32", _seq_fp32(a, w, b), a, w, b)
    e, _ = _ref64(a, w, b)
    a_drop = a.clone()
    a_drop[:, 640:704] = 0
    defects = {"k-block dropped": _ref64(a_drop, w, b)[0].to(BF16), "bias omitted": _ref64(a, w, None)[0].to(BF16)}
    shifted = e.to(BF16).clone()
    shifted[:, 16:24] = e[:, 24:32].to(BF16)
    defects["column group shifted"] = shifted
    for name, wrong in defects.items():
        with pytest.raises(AssertionError):
            check_bound(f"self-check {name}", wrong, a, w, b)
