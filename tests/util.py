"""Shared helpers of the parity tests."""
import json
import os

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")

# BASELINE.json north_star tolerance
RTOL, ATOL = 1e-3, 1e-5


def gold(name):
    return np.load(os.path.join(GOLD, name + ".npz"))


def t(a, device=None, dtype=None):
    x = torch.from_numpy(np.ascontiguousarray(a))
    if dtype is not None:
        x = x.to(dtype)
    return x.to(device) if device is not None else x


def check_close(actual, expected, what, rtol=RTOL, atol=ATOL, scale_atol=True, max_strict_viol=1e-4):
    """Parity check used by every floating-point test.

    * hard bound: |a - e| <= atol_eff + rtol * |e| everywhere, atol_eff = atol * max(1, max|e|):
      fp32 recurrences of length L accumulate an ABSOLUTE error proportional to the magnitude of the
      summands (two faithful fp32 CPU implementations -- the reference's selective_scan_ref and the C
      restatement -- differ by 4e-4 at max|out| = 407 on BASELINE config 1), so the absolute floor
      scales with the output range;
    * strict bound: the fraction of elements violating the UNSCALED north-star tolerance
      (rtol 1e-3, atol 1e-5) must stay below max_strict_viol (default 1e-4; measured on BASELINE
      config 1: 7.6e-7 between the two CPU fp32 implementations, 3.2e-5 for the sm_90a kernel
      whose exp2/log2/rcp are MUFU approximations of ~2^-22 relative error).
    """
    a = torch.as_tensor(actual).detach().float().cpu()
    e = torch.as_tensor(expected).detach().float().cpu()
    assert a.shape == e.shape, f"{what}: shape {tuple(a.shape)} vs {tuple(e.shape)}"
    assert torch.isfinite(a).all(), f"{what}: non-finite values in result"
    diff = (a - e).abs()
    emax = e.abs().max().item() if e.numel() else 0.0
    atol_eff = atol * max(1.0, emax) if scale_atol else atol
    bad = diff > (atol_eff + rtol * e.abs())
    strict = (diff > (atol + rtol * e.abs())).float().mean().item() if e.numel() else 0.0
    msg = (f"{what}: max|diff|={diff.max().item() if e.numel() else 0:.3e} max|ref|={emax:.3e} "
           f"viol(hard)={int(bad.sum())}/{e.numel()} strict_viol_frac={strict:.2e}")
    print("   ", msg)
    _log_parity(what, diff.max().item() if e.numel() else 0.0, emax, strict, int(bad.sum()), e.numel(), rtol, atol, max_strict_viol)
    assert not bad.any(), msg
    assert strict <= max_strict_viol, msg + f" (strict fraction > {max_strict_viol})"


def _log_parity(what, max_diff, max_ref, strict, hard_viol, numel, rtol, atol, max_strict_viol):
    """With ZIGMA_PARITY_LOG=<file> in the environment, appends the achieved error of every check to that JSON-lines file, so
    the numbers behind "N passed" survive the run.  Nothing is written otherwise (the source tree may be read-only)."""
    path = os.environ.get("ZIGMA_PARITY_LOG")
    if not path:
        return
    try:
        rec = dict(test=os.environ.get("PYTEST_CURRENT_TEST", "").split(" ")[0], what=what, max_diff=max_diff, max_ref=max_ref,
                   strict_viol_frac=strict, hard_viol=hard_viol, numel=numel, rtol=rtol, atol=atol, max_strict_viol=max_strict_viol)
        with open(path, "a") as f:
            f.write(json.dumps(rec) + "\n")
    except OSError:
        pass


# ------------------------------------------------------------------------------------------------ bounds against fp64 references
# Shared by the kernel-against-fp64 files (test_gpu_norm_kernels.py, test_gpu_scan_kernels.py).  a: kernel output; e: the fp64
# reference before the output's final rounding; M: the fp64 magnitude of the terms that form each element (never |e|, which is
# small exactly where the terms cancel); S: the sum of |term| over what a reduced output sums.
MANT = {torch.float16: 10, torch.bfloat16: 7, torch.float32: 23}
DTYPE_NAME = {torch.float32: "fp32", torch.float16: "fp16", torch.bfloat16: "bf16"}
C_F32 = 64                                  # fp32 elements: |a - e| <= c_f32 * 2^-24 * M (+ the smallest normal fp32)
COLSUM_REL = 1e-5                           # sums: |a - e| <= rel * S + one ulp of the returned dtype
MISMATCH = {torch.float16: 5e-3, torch.bfloat16: 1e-3}      # 16-bit: fraction of elements that differ from round(e)


def ulp(e, dtype):
    """Unit in the last place of `dtype` at the fp64 values e (the subnormal spacing below the normal range)."""
    _, ex = torch.frexp(e.abs())
    u = torch.ldexp(torch.ones_like(e), ex - 1 - MANT[dtype])
    floor = torch.finfo(dtype).tiny * 2.0 ** -MANT[dtype]
    return torch.where(e == 0, torch.full_like(e, floor), u.clamp(min=floor))


def _log(what, dtype, **rec):
    path = os.environ.get("ZIGMA_PARITY_LOG")
    if path:
        rec = dict(test=os.environ.get("PYTEST_CURRENT_TEST", "").split(" ")[0], what=what, dtype=DTYPE_NAME[dtype], **rec)
        with open(path, "a") as f:
            f.write(json.dumps(rec) + "\n")


def check_elem(what, a, e, M, max_ulp=1, extra=None, c_f32=C_F32, mismatch=None, conditioned=False):
    """Elementwise bound.  fp32: |a - e| <= c_f32 * 2^-24 * M + the smallest normal fp32 (a result that underflows may flush).
    16-bit: at most max_ulp ulps of e, or, for an element formed by cancellation, the fp32 bound plus one ulp (plus `extra`:
    what a one-ulp difference of a rounded intermediate that is not an output moves the element by); and the fraction of
    elements that differ from round(e) stays below mismatch (default MISMATCH[dtype]); conditioned: among the elements whose
    fp32 allowance is under a quarter ulp only."""
    dtype = a.dtype
    a = a.detach().double().to(e.device)
    assert a.shape == e.shape, f"{what}: shape {tuple(a.shape)} vs {tuple(e.shape)}"
    assert torch.isfinite(a).all(), f"{what}: non-finite values"
    diff = (a - e).abs()
    fp32_bound = c_f32 * 2.0 ** -24 * M + torch.finfo(torch.float32).tiny
    c = (diff / M.clamp(min=1e-300) / 2.0 ** -24).max().item() if a.numel() else 0.0
    if dtype == torch.float32:
        bad = diff > fp32_bound
        _log(what, dtype, worst_c=c, frac_of_bound=(diff / fp32_bound).max().item() if a.numel() else 0.0, numel=a.numel())
        assert not bad.any(), f"{what}: {int(bad.sum())}/{a.numel()} beyond {c_f32}*2^-24*M (worst c {c:.1f})"
        return
    u = ulp(e, dtype)
    dist = diff / u
    allow = torch.maximum(max_ulp * u, fp32_bound + u + (0 if extra is None else extra))
    bad = diff > allow
    # the mismatch fraction counts the elements whose fp32 allowance is under a quarter ulp (or all, conditioned=False): where
    # long accumulation or cancellation makes M large against |e|, a differing last bit says nothing about a rounding point
    cond = (fp32_bound <= 0.25 * u) if conditioned else torch.ones_like(u, dtype=torch.bool)
    mism = (a != e.to(dtype).double())[cond].double().mean().item() if cond.any() else 0.0
    worst = dist.max().item() if a.numel() else 0.0
    _log(what, dtype, max_ulp=worst, frac_of_bound=(diff / allow).max().item() if a.numel() else 0.0, mismatch_frac=mism, numel=a.numel())
    assert not bad.any(), f"{what}: {int(bad.sum())}/{a.numel()} elements beyond {max_ulp} ulp (worst {worst:.2f} ulp)"
    limit = MISMATCH[dtype] if mismatch is None else mismatch
    assert mism <= limit, f"{what}: {mism:.2e} of the elements differ from the rounded reference"


def check_colsum(what, a, e, S, rel=COLSUM_REL):
    """Reduced outputs (weight / bias / modulation gradients, sums over rows or channels): |a - e| <= rel * S + one ulp
    (+ the smallest normal fp32)."""
    dtype = a.dtype
    ad = a.detach().double().to(e.device)
    assert ad.shape == e.shape and torch.isfinite(ad).all(), what
    bound = rel * S + ulp(e, dtype) + torch.finfo(torch.float32).tiny     # (fp32 accumulation flushes subnormal terms)
    worst = ((ad - e).abs() / bound).max().item() if ad.numel() else 0.0
    _log(what, dtype, colsum_worst_frac_of_bound=worst, numel=ad.numel())
    assert worst <= 1.0, f"{what}: sum off by {worst:.2f} x ({rel:g} S + 1 ulp)"


def model_case(name):
    g = gold("model_" + name)
    cfg = json.loads(bytes(g["cfg_json"]).decode())
    shapes = json.loads(bytes(g["shapes_json"]).decode())
    return g, cfg, {k: tuple(v) for k, v in shapes.items()}
