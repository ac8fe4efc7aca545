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


def model_case(name):
    g = gold("model_" + name)
    cfg = json.loads(bytes(g["cfg_json"]).decode())
    shapes = json.loads(bytes(g["shapes_json"]).decode())
    return g, cfg, {k: tuple(v) for k, v in shapes.items()}
