"""BENCH/TEST INFRASTRUCTURE -- the reference's OWN compiled CUDA kernels (oracle/_ref/*.so, built
from the unmodified sources under /root/reference by oracle/build_ref.sh, gencode swapped to
sm_90a) behind the restated glue of oracle/zigma_oracle.py: the "reference vendored CUDA path"
baseline that BASELINE.md section 5 asks to time on the same box.  Never imported by the product
package; bench.py uses it only to report the baseline next to our numbers.

Glue = what the reference's Python does around its kernels (channel-first layout, index_select
permutation + .contiguous(), separate x_proj / dt_proj GEMMs, rearranged contiguous B/C, unfused
modulate / gate), restated in zigma_oracle.py and pinned against the reference there.  The one
substitution: the reference's Triton add+RMSNorm kernel cannot travel (Python source), so the
baseline borrows OUR fused add+norm kernel for that op -- this can only flatter the baseline.
"""
import importlib.util
import os
import sys

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
_REF = os.path.join(_HERE, "_ref")
_mods = {}


def available():
    return all(os.path.exists(os.path.join(_REF, n + ".so")) for n in ("selective_scan_cuda", "causal_conv1d_cuda"))


def load():
    if not _mods:
        for name in ("selective_scan_cuda", "causal_conv1d_cuda"):
            spec = importlib.util.spec_from_file_location(name, os.path.join(_REF, name + ".so"))
            mod = importlib.util.module_from_spec(spec)
            spec.loader.exec_module(mod)
            _mods[name] = mod
    return _mods["selective_scan_cuda"], _mods["causal_conv1d_cuda"]


def scan_fwd(u, delta, A, B, C, D, z, delta_bias, delta_softplus=True):
    """selective_scan_cuda.fwd (selective_scan.cpp:226-336): returns out_z (or out when z is None)."""
    ss, _ = load()
    if B.dim() == 3:
        B, C = B.unsqueeze(1), C.unsqueeze(1)
    res = ss.fwd(u, delta, A, B.contiguous(), C.contiguous(), D, z, delta_bias, delta_softplus)
    return res[-1] if z is not None else res[0]


def conv_fwd(x, w, b, silu=True):
    _, cc = load()
    return cc.causal_conv1d_fwd(x, w, b, silu)


def backend(norm_fn=None):
    """BACKEND dict for zigma_oracle: reference CUDA kernels (+ our norm kernel, see module doc)."""
    be = {"conv": lambda x, w, b: conv_fwd(x, w.contiguous(), b, True),
          "scan": lambda u, d, A, B, C, D, z, bias: scan_fwd(u, d, A, B, C, D, z, bias, True)}
    if norm_fn is not None:
        be["norm"] = norm_fn
    return be


# ---- training: the reference kernels' forward AND backward behind autograd -----------------------------
class _RefScanFn(torch.autograd.Function):
    """selective_scan_cuda.fwd / .bwd the way SelectiveScanFn drives them (selective_scan_interface.py:21-83)."""

    @staticmethod
    def forward(ctx, u, delta, A, B, C, D, z, delta_bias):
        ss, _ = load()
        if B.dim() == 3:
            B, C = B.unsqueeze(1), C.unsqueeze(1)
            ctx.squeeze = True
        else:
            ctx.squeeze = False
        B, C = B.contiguous(), C.contiguous()
        if u.stride(-1) != 1:
            u = u.contiguous()
        if delta.stride(-1) != 1:
            delta = delta.contiguous()
        if z is not None and z.stride(-1) != 1:
            z = z.contiguous()
        res = ss.fwd(u, delta, A, B, C, D, z, delta_bias, True)
        out, x = res[0], res[1]
        ctx.save_for_backward(u, delta, A, B, C, D, z, delta_bias, x, out)
        return res[-1] if z is not None else out

    @staticmethod
    def backward(ctx, dout):
        ss, _ = load()
        u, delta, A, B, C, D, z, delta_bias, x, out = ctx.saved_tensors
        if dout.stride(-1) != 1:
            dout = dout.contiguous()
        r = ss.bwd(u, delta, A, B, C, D, z, delta_bias, dout, x, out, None, True, False)
        du, ddelta, dA, dB, dC, dD, dbias = r[:7]
        dz = r[7] if z is not None else None
        if ctx.squeeze:
            dB, dC = dB.squeeze(1), dC.squeeze(1)
        return du, ddelta, dA, dB.to(B.dtype), dC.to(C.dtype), dD, dz, dbias


class _RefConvFn(torch.autograd.Function):
    """causal_conv1d_fwd / _bwd (causal_conv1d_interface.py:11-47)."""

    @staticmethod
    def forward(ctx, x, w, b):
        _, cc = load()
        if x.stride(2) != 1 and x.stride(1) != 1:
            x = x.contiguous()
        ctx.save_for_backward(x, w, b)
        return cc.causal_conv1d_fwd(x, w, b, True)

    @staticmethod
    def backward(ctx, dout):
        _, cc = load()
        x, w, b = ctx.saved_tensors
        if dout.stride(2) != 1 and dout.stride(1) != 1:
            dout = dout.contiguous()
        dx, dw, db = cc.causal_conv1d_bwd(x, w, b, dout, None, True)
        return dx, dw, db


def train_backend(norm_fn=None):
    """BACKEND for zigma_oracle under autograd: reference CUDA forward + backward kernels."""
    be = {"conv": lambda x, w, b: _RefConvFn.apply(x, w.contiguous(), b),
          "scan": lambda u, d, A, B, C, D, z, bias: _RefScanFn.apply(u, d, A, B, C, D, z, bias)}
    if norm_fn is not None:
        be["norm"] = norm_fn
    return be
