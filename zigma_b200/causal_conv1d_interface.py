"""Host-side mirror of ``dis_causal_conv1d/causal_conv1d/causal_conv1d_interface.py`` (reference)
over the sm_90a kernels: ``causal_conv1d_fn`` (:37-46) with its autograd Function (:10-34).
``causal_conv1d_update`` (single-token decode, :68-80) is out of scope: diffusion sampling never
decodes autoregressively (SURVEY.md section 2 #4)."""
import torch

from . import _lib


def _conv_fwd(x, weight, bias, silu, x_rowmap=None, out=None, seg_len=0):
    """causal_conv1d_cuda.causal_conv1d_fwd (causal_conv1d.cpp:130-189).  x: logical
    (batch, dim, seqlen) with stride(2) == 1 (channel first) or stride(1) == 1 (channel last)."""
    _lib.require_cuda(x, weight, bias)
    if x.dim() != 3:
        raise RuntimeError("causal_conv1d: x must be (batch, dim, seqlen)")
    batch, dim, seqlen = x.shape
    if weight.dim() != 2 or weight.shape[0] != dim:
        raise RuntimeError("causal_conv1d: weight must be (dim, width)")
    width = weight.shape[1]
    if not 2 <= width <= 4:
        raise RuntimeError("causal_conv1d only supports width between 2 and 4")
    if bias is not None and (bias.shape != (dim,) or bias.dtype != weight.dtype):
        raise RuntimeError("causal_conv1d: bias must be (dim,) with the dtype of weight")
    if x.stride(2) != 1 and x.stride(1) != 1:
        x = x.contiguous()
    channel_last = x.stride(2) != 1 and seqlen != 1
    weight = weight.contiguous()
    bias = bias.contiguous() if bias is not None else None
    if out is None:
        if channel_last:
            out = torch.empty((batch, seqlen, dim), dtype=x.dtype, device=x.device).transpose(1, 2)
        else:
            out = torch.empty((batch, dim, seqlen), dtype=x.dtype, device=x.device)
    p = _lib.ConvParams()
    p.x, p.weight, p.bias, p.out = _lib.ptr(x), _lib.ptr(weight), _lib.ptr(bias), _lib.ptr(out)
    p.x_rowmap = _lib.ptr(x_rowmap)
    p.x_sb, p.x_sd, p.x_sl = x.stride()
    p.out_sb, p.out_sd, p.out_sl = out.stride()
    if seqlen == 1:
        p.x_sl = p.out_sl = 1
    p.batch, p.dim, p.seqlen, p.width = batch, dim, seqlen, width
    p.dtype, p.wdtype, p.silu = _lib.dt(x), _lib.dt(weight), int(bool(silu))
    p.seg_len = int(seg_len)       # independent segments of this length inside the sequence (temporal video scan), 0 = one sequence
    _lib.call("zg_causal_conv1d_fwd", p)
    return out


def _conv_bwd(x, weight, bias, dout, silu, dx_out=None, x_rowmap=None):
    """causal_conv1d_cuda.causal_conv1d_bwd (causal_conv1d.cpp:191-268): returns dx, dweight (fp32),
    dbias (fp32 or None).  Channel-first tensors (stride(2) == 1; a provided dx_out is written in
    place -- the reference uses that to fill one half of dxz, selective_scan_interface.py:425-427) or
    token-major ones (stride(1) == 1, all three of x / dout / dx), where ``x_rowmap`` (int32, seqlen)
    says the conv ran over the gathered sequence x[:, :, x_rowmap]: x is read and dx written through it."""
    batch, dim, seqlen = x.shape
    tok = x.stride(1) == 1 and not (x.stride(2) == 1 and dim > 1) and seqlen > 1
    if tok:
        if dout.stride(1) != 1:
            dout = dout.transpose(1, 2).contiguous().transpose(1, 2)
        dx = dx_out if dx_out is not None else torch.empty((batch, seqlen, dim), dtype=x.dtype, device=x.device).transpose(1, 2)
        if dx.stride(1) != 1:
            raise RuntimeError("causal_conv1d_bwd: dx must be token-major like x")
    else:
        if x_rowmap is not None:
            raise RuntimeError("causal_conv1d_bwd: x_rowmap needs token-major (dim-contiguous) tensors")
        if x.stride(2) != 1:
            x = x.contiguous()
        if dout.stride(2) != 1:
            dout = dout.contiguous()
        dx = dx_out if dx_out is not None else torch.empty_like(x, memory_format=torch.contiguous_format)
        if dx.stride(2) != 1:
            raise RuntimeError("causal_conv1d_bwd: dx must have seq stride 1")
    weight = weight.contiguous()
    dweight = torch.zeros(weight.shape, dtype=torch.float32, device=x.device)
    dbias = torch.zeros((dim,), dtype=torch.float32, device=x.device) if bias is not None else None
    q = _lib.ConvBwdParams()
    p = q.fwd
    p.x, p.weight, p.bias = _lib.ptr(x), _lib.ptr(weight), _lib.ptr(bias)
    p.x_rowmap = _lib.ptr(x_rowmap)
    p.x_sb, p.x_sd, p.x_sl = x.stride()
    p.batch, p.dim, p.seqlen, p.width = batch, dim, seqlen, weight.shape[1]
    p.dtype, p.wdtype, p.silu = _lib.dt(x), _lib.dt(weight), int(bool(silu))
    q.dout, q.dx, q.dweight, q.dbias = _lib.ptr(dout), _lib.ptr(dx), _lib.ptr(dweight), _lib.ptr(dbias)
    q.dout_sb, q.dout_sd, q.dout_sl = dout.stride()
    q.dx_sb, q.dx_sd, q.dx_sl = dx.stride()
    if not tok:
        p.x_sl = q.dout_sl = q.dx_sl = 1           # (seqlen == 1: any stride is "contiguous")
    # `out` only takes part in the shared validation (layout class of the call)
    p.out = _lib.ptr(dx)
    p.out_sb, p.out_sd, p.out_sl = q.dx_sb, q.dx_sd, q.dx_sl
    _lib.call_bwd("zg_causal_conv1d_bwd", q)
    return dx, dweight, dbias


class CausalConv1dFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, weight, bias=None, activation=None):
        if activation not in [None, "silu", "swish"]:
            raise NotImplementedError("activation must be None, silu, or swish")
        ctx.save_for_backward(x, weight, bias)
        ctx.activation = activation in ["silu", "swish"]
        return _conv_fwd(x, weight, bias, ctx.activation)

    @staticmethod
    def backward(ctx, dout):
        x, weight, bias = ctx.saved_tensors
        dx, dweight, dbias = _conv_bwd(x, weight, bias, dout, ctx.activation)
        if dx.shape != x.shape:
            dx = dx.reshape(x.shape)
        return dx, dweight.to(weight.dtype), (dbias.to(bias.dtype) if bias is not None else None), None


def causal_conv1d_fn(x, weight, bias=None, activation=None):
    """x: (batch, dim, seqlen); weight: (dim, width); bias: (dim,); activation: None | "silu" | "swish".
    out: (batch, dim, seqlen)."""
    return CausalConv1dFn.apply(x, weight, bias, activation)
