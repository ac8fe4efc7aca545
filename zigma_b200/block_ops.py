"""The elementwise part of a ZigMa block under autograd, fused (training counterpart of the engine's block tail):

    hidden   = x + gate * mix[:, rowmap]       the previous block's gated residual add + un-permutation (model_zigma.py:445)
    r        = residual + hidden               fused add ...
    normed   = RMSNorm(r) * norm_w             ... + norm (layernorm.py:64-120), prenorm, fp32 residual stream
    modded   = normed * (1 + scale) + shift    adaLN modulate (model_zigma.py:60-62)

Forward: ``zg_block_tail_fwd`` (one pass, the reference's bf16 rounding points replicated); backward:
``zg_block_tail_bwd`` (one pass: RMSNorm backward, d_mix scattered back to scan order, dgate / dshift / dscale /
d_norm_w column sums in registers).  The unfused graph costs ~12 elementwise / reduction kernels per block and
direction (DESIGN.md section 4.4).
"""
import torch

from . import _lib
from .engine import block_tail


def _contig(t):
    return None if t is None else (t if t.is_contiguous() else t.contiguous())


def tail_bwd_nparts(batch, seqlen, sms):
    """CTAs of zg_block_tail_bwd, which are also the rows of its d_norm_w partials buffer: about one per 64 token rows, at
    most 3 per SM, and at least one warp (4 per CTA) per batch element, which the deterministic kernel needs.  The atomic
    and the deterministic kernel get the same value, so their d_norm_w partial rows have the same layout."""
    nparts = max(1, min((batch * seqlen + 63) // 64, 3 * sms), (batch + 3) // 4)
    if nparts > 65535:
        raise RuntimeError(f"block_tail_fn backward: batch {batch} needs {nparts} CTAs, more than the 65535 the kernel takes")
    return nparts


class BlockTailFn(torch.autograd.Function):
    """(x, mix, gate, shift, scale, norm_w, residual, rowmap, eps, path_scale) -> (residual_out fp32, normed, modded).
    x, mix: (B, L, D) contiguous; gate / shift / scale: (B, D) views with one common row stride (chunks of adaLN's
    (B, 3D) output); residual: (B, L, D) fp32 or None; rowmap: int32 (L,) or None; mix / gate None for the first block.
    path_scale: None, or the block's drop-path multipliers (B,) in x.dtype (stochastic depth in training): the hidden
    state joins the residual as hidden * path_scale[b] (zg_block_tail_fwd_dp / _bwd_dp); it gets no gradient."""

    @staticmethod
    def forward(ctx, x, mix, gate, shift, scale, norm_w, residual, rowmap, eps, path_scale=None):
        x, mix, residual = _contig(x), _contig(mix), _contig(residual)
        # one dtype for every operand of the kernels (x's): see engine.block_tail.  The casts happen HERE so that the
        # tensors saved for the backward are the ones the forward kernel actually read.
        ctx.in_dtypes = tuple(None if t is None else t.dtype for t in (mix, gate, shift, scale))
        cast = lambda t: t if (t is None or t.dtype == x.dtype) else t.to(x.dtype)
        mix, gate, shift, scale = cast(mix), cast(gate), cast(shift), cast(scale)
        mods = [m for m in (gate, shift, scale) if m is not None]
        if mods and any(m.stride(0) != mods[0].stride(0) or m.stride(1) != 1 for m in mods):
            gate, shift, scale = [None if m is None else m.contiguous() for m in (gate, shift, scale)]
        res_out, normed, modded, rstd = block_tail(x, mix, gate, shift, scale, norm_w, residual, rowmap, eps, want_rstd=True,
                                                   path_scale=path_scale)
        ctx.save_for_backward(res_out, rstd, mix, gate, scale, norm_w, rowmap, path_scale)
        ctx.has_res = residual is not None
        return res_out, normed, modded

    @staticmethod
    def backward(ctx, d_res_out, d_normed, d_modded):
        res_out, rstd, mix, gate, scale, norm_w, rowmap, path_scale = ctx.saved_tensors
        B, L, D = res_out.shape
        act = scale.dtype
        dev = res_out.device
        d_res_out, d_normed, d_modded = _contig(d_res_out), _contig(d_normed), _contig(d_modded)
        d_x = torch.empty((B, L, D), dtype=act, device=dev)
        d_mix = torch.empty((B, L, D), dtype=act, device=dev) if mix is not None else None
        d_res_in = torch.empty((B, L, D), dtype=torch.float32, device=dev) if ctx.has_res else None
        acc = torch.zeros((3, B, D), dtype=torch.float32, device=dev)
        nparts = tail_bwd_nparts(B, L, torch.cuda.get_device_properties(dev).multi_processor_count)
        d_w = torch.empty((nparts, D), dtype=torch.float32, device=dev)       # per-CTA partial sums, added up below
        nw = norm_w if norm_w.dtype == act else norm_w.to(act)
        q = _lib.BlockTailBwdParams()
        q.d_residual_out, q.d_normed, q.d_modded = _lib.ptr(d_res_out), _lib.ptr(d_normed), _lib.ptr(d_modded)
        q.r, q.rstd, q.mix, q.gate, q.scale, q.norm_w, q.rowmap = (_lib.ptr(res_out), _lib.ptr(rstd), _lib.ptr(mix), _lib.ptr(gate),
                                                                   _lib.ptr(scale), _lib.ptr(nw), _lib.ptr(rowmap))
        q.d_x, q.d_mix, q.d_residual_in = _lib.ptr(d_x), _lib.ptr(d_mix), _lib.ptr(d_res_in)
        q.dgate, q.dshift, q.dscale, q.d_norm_w = (_lib.ptr(acc[0]) if mix is not None else None), _lib.ptr(acc[1]), _lib.ptr(acc[2]), _lib.ptr(d_w)
        q.mod_rs = scale.stride(0)
        q.batch, q.seqlen, q.dim, q.dtype, q.nparts = B, L, D, _lib.dt(act), nparts
        if path_scale is None:
            _lib.call_bwd("zg_block_tail_bwd", q)
        else:
            _lib.call_bwd("zg_block_tail_bwd_dp", _lib.BlockTailBwdDpParams(q, _lib.ptr(path_scale)))
        dt_mix, dt_gate, dt_shift, dt_scale = ctx.in_dtypes
        return (d_x, None if d_mix is None else d_mix.to(dt_mix), acc[0].to(dt_gate) if mix is not None else None,
                acc[1].to(dt_shift or act), acc[2].to(dt_scale or act), d_w.sum(0).to(norm_w.dtype), d_res_in, None, None, None)


def block_tail_fn(x, mix, gate, shift, scale, norm_w, residual, rowmap, eps, path_scale=None):
    return BlockTailFn.apply(x, mix, gate, shift, scale, norm_w, residual, rowmap, eps, path_scale)
