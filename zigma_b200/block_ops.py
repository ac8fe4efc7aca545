"""The elementwise part of a ZigMa block under autograd, fused (training counterpart of the engine's block tail):

    hidden   = x + gate * mix[:, rowmap]       the previous block's gated residual add + un-permutation (model_zigma.py:445)
    r        = residual + hidden               fused add ...
    normed   = RMSNorm(r) * norm_w             ... + norm (layernorm.py:64-120), prenorm, fp32 residual stream
    modded   = normed * (1 + scale) + shift    adaLN modulate (model_zigma.py:60-62)

Forward: ``zg_block_tail_fwd`` (one pass, the reference's bf16 rounding points replicated); backward:
``zg_block_tail_bwd`` (one pass: RMSNorm backward, d_mix scattered back to scan order, dgate / dshift / dscale /
d_norm_w column sums in registers).  The unfused graph costs ~12 elementwise / reduction kernels per block and
direction (DESIGN.md section 4.4).

TextPrologueFn is the text branch of a has_text block up to the cross-attention (model_zigma.py:206-208):

    hidden   = x + gate * mix[:, rowmap]                          the mixer's gated residual add + un-permutation
    q_in     = LayerNorm_noaffine(hidden) * (1 + scale) + shift    norm_msa + modulate

on ``zg_text_prologue_fwd`` / ``zg_text_prologue_bwd`` (DESIGN.md section 4.7).
"""
import torch

from . import _lib
from .engine import block_tail, text_prologue


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


class TextPrologueFn(torch.autograd.Function):
    """(x, mix, gate, rowmap, shift, scale, eps) -> (hidden, q_in).  x, mix: (B, L, D) (mix in scan order, rowmap: int32 (L,)
    or None); gate / shift / scale: (B, D) views (chunks of adaLN's output).  Every operand is brought to x.dtype, the
    casting policy of BlockTailFn; hidden and q_in are in x.dtype.  The backward runs zg_text_prologue_bwd (its _det twin
    under torch.use_deterministic_algorithms)."""

    @staticmethod
    def forward(ctx, x, mix, gate, rowmap, shift, scale, eps):
        x, mix = _contig(x), _contig(mix)
        ctx.in_dtypes = (mix.dtype, gate.dtype, shift.dtype, scale.dtype)
        cast = lambda t: t if t.dtype == x.dtype else t.to(x.dtype)
        mix, gate, shift, scale = cast(mix), cast(gate), cast(shift), cast(scale)
        if any(m.stride(0) != gate.stride(0) or m.stride(1) != 1 for m in (gate, shift, scale)):
            gate, shift, scale = gate.contiguous(), shift.contiguous(), scale.contiguous()
        hidden, q_in, mean, rstd = text_prologue(x, mix, gate, shift, scale, rowmap, eps, want_stats=True)
        ctx.save_for_backward(hidden, mean, rstd, mix, gate, scale, rowmap)
        return hidden, q_in

    @staticmethod
    def backward(ctx, d_hidden, d_q):
        hidden, mean, rstd, mix, gate, scale, rowmap = ctx.saved_tensors
        B, L, D = hidden.shape
        act, dev = hidden.dtype, hidden.device
        if d_q is None:
            d_q = torch.zeros_like(hidden)
        d_hidden, d_q = _contig(d_hidden), _contig(d_q)
        d_x, d_mix = torch.empty_like(hidden), torch.empty_like(hidden)
        acc = torch.zeros((3, B, D), dtype=torch.float32, device=dev)
        q = _lib.TextPrologueBwdParams()
        q.d_hidden, q.d_q, q.hidden, q.mix, q.gate, q.scale = (_lib.ptr(d_hidden), _lib.ptr(d_q), _lib.ptr(hidden), _lib.ptr(mix),
                                                               _lib.ptr(gate), _lib.ptr(scale))
        q.mean, q.rstd, q.rowmap, q.d_x, q.d_mix = _lib.ptr(mean), _lib.ptr(rstd), _lib.ptr(rowmap), _lib.ptr(d_x), _lib.ptr(d_mix)
        q.dgate, q.dshift, q.dscale = _lib.ptr(acc[0]), _lib.ptr(acc[1]), _lib.ptr(acc[2])
        q.mod_rs = gate.stride(0)
        q.batch, q.seqlen, q.dim, q.dtype = B, L, D, _lib.dt(act)
        q.nparts = tail_bwd_nparts(B, L, torch.cuda.get_device_properties(dev).multi_processor_count)
        _lib.call_bwd("zg_text_prologue_bwd", q)
        dt_mix, dt_gate, dt_shift, dt_scale = ctx.in_dtypes
        return d_x, d_mix.to(dt_mix), acc[0].to(dt_gate), None, acc[1].to(dt_shift), acc[2].to(dt_scale), None


def text_prologue_fn(x, mix, gate, rowmap, shift, scale, eps):
    return TextPrologueFn.apply(x, mix, gate, rowmap, shift, scale, eps)
