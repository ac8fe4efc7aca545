"""Host-side mirror of ``dis_mamba/mamba_ssm/ops/triton/layernorm.py`` (reference) over hand-written
sm_90a kernels -- the reference launches Triton here; north_star forbids Triton on the hot path.
``rms_norm_fn`` (:477-478), ``layer_norm_fn`` (:464-474), ``RMSNorm`` (:481-503), ``LayerNormFn``
(:380-461)."""
import torch

from . import _lib


def _norm_fwd(x, weight, bias, eps, residual, residual_dtype, is_rms):
    """_layer_norm_fwd (layernorm.py:123-177) on a 2-D view.  Returns y, mean, rstd, residual_out."""
    M, N = x.shape
    y = torch.empty_like(x, memory_format=torch.contiguous_format)
    if residual is not None:
        residual_dtype = residual.dtype
    store_res = residual is not None or (residual_dtype is not None and residual_dtype != x.dtype)
    res_out = torch.empty((M, N), dtype=residual_dtype, device=x.device) if store_res else None
    mean = torch.empty((M,), dtype=torch.float32, device=x.device) if not is_rms else None
    rstd = torch.empty((M,), dtype=torch.float32, device=x.device)
    p = _lib.NormParams()
    p.x, p.residual, p.weight, p.bias = _lib.ptr(x), _lib.ptr(residual), _lib.ptr(weight), _lib.ptr(bias)
    p.y, p.residual_out, p.mean, p.rstd = _lib.ptr(y), _lib.ptr(res_out), _lib.ptr(mean), _lib.ptr(rstd)
    p.x_rs, p.y_rs = x.stride(0), y.stride(0)
    p.res_rs = residual.stride(0) if residual is not None else 0
    p.resout_rs = res_out.stride(0) if res_out is not None else 0
    p.nrows, p.ncols = M, N
    p.dtype = _lib.dt(x)
    p.res_dtype = _lib.dt(residual_dtype) if store_res else p.dtype
    p.wdtype = _lib.dt(weight) if weight is not None else p.dtype
    p.is_rms, p.eps = int(is_rms), float(eps)
    _lib.call("zg_add_norm_fwd", p)
    return y, mean, rstd, (res_out if res_out is not None else x)


def _norm_bwd(dy, x, weight, bias, mean, rstd, dresidual, has_residual, is_rms, x_dtype):
    """_layer_norm_bwd (layernorm.py:293-377)."""
    M, N = x.shape
    dx = torch.empty((M, N), dtype=x_dtype, device=x.device)
    dres_in = torch.empty_like(x) if (has_residual and dx.dtype != x.dtype) else None
    dw = torch.zeros((N,), dtype=torch.float32, device=x.device) if weight is not None else None
    db = torch.zeros((N,), dtype=torch.float32, device=x.device) if bias is not None else None
    p = _lib.NormBwdParams()
    p.dy, p.dresidual, p.x, p.weight = _lib.ptr(dy), _lib.ptr(dresidual), _lib.ptr(x), _lib.ptr(weight)
    p.mean, p.rstd, p.dx, p.dresidual_in = _lib.ptr(mean), _lib.ptr(rstd), _lib.ptr(dx), _lib.ptr(dres_in)
    p.dweight, p.dbias = _lib.ptr(dw), _lib.ptr(db)
    p.dy_rs, p.x_rs, p.dx_rs = dy.stride(0), x.stride(0), dx.stride(0)
    p.dres_rs = dresidual.stride(0) if dresidual is not None else 0
    p.dresin_rs = dres_in.stride(0) if dres_in is not None else 0
    p.nrows, p.ncols = M, N
    p.dtype, p.res_dtype = _lib.dt(x_dtype), _lib.dt(x)
    p.wdtype = _lib.dt(weight) if weight is not None else p.dtype
    p.is_rms = int(is_rms)
    if dy.dtype != x_dtype:
        dy = dy.to(x_dtype)
        p.dy, p.dy_rs = _lib.ptr(dy), dy.stride(0)
    _lib.call_bwd("zg_add_norm_bwd", p)
    if has_residual and dx.dtype == x.dtype:
        dres_in = dx
    return dx, (dw.to(weight.dtype) if dw is not None else None), (db.to(bias.dtype) if db is not None else None), dres_in


def _rows(t):
    """(…, N) -> (M, N) with a unit inner stride (a view whenever the memory allows it)."""
    t2 = t.reshape(-1, t.shape[-1])
    return t2 if t2.stride(-1) == 1 else t2.contiguous()


class LayerNormFn(torch.autograd.Function):
    """Autograd node of the fused (residual add +) LayerNorm / RMSNorm.  Contract of the reference's node of the same name
    (dis_mamba/mamba_ssm/ops/triton/layernorm.py:380-461): inputs (x, weight, bias, residual, eps, prenorm, residual_in_fp32,
    is_rms_norm); output y, or (y, residual_out) with prenorm; gradients for x, weight, bias, residual.  The body is this
    repo's: everything is flattened to rows once, the saved state is the kernel's own outputs (the summed residual stream r,
    mean, rstd), and the backward feeds zg_add_norm_bwd, which produces dx and the residual gradient in one pass."""

    @staticmethod
    def forward(ctx, x, weight, bias, residual=None, eps=1e-6, prenorm=False, residual_in_fp32=False, is_rms_norm=False):
        _lib.require_cuda(x, weight, bias, residual)
        shape = x.shape
        if residual is not None and residual.shape != shape:
            raise RuntimeError(f"layer_norm_fn: residual shape {tuple(residual.shape)} != input shape {tuple(shape)}")
        x2 = _rows(x)
        r2 = None if residual is None else _rows(residual)
        # dtype of the residual stream the kernel writes: the incoming stream's, else fp32 on request, else "same as x" (not stored)
        stream_dtype = r2.dtype if r2 is not None else (torch.float32 if residual_in_fp32 else None)
        y, mean, rstd, stream = _norm_fwd(x2, weight.contiguous(), None if bias is None else bias.contiguous(), eps, r2, stream_dtype, is_rms_norm)
        ctx.save_for_backward(stream, weight, bias, mean, rstd)
        ctx.meta = (shape, x2.dtype, bool(is_rms_norm), residual is not None, bool(prenorm))
        y = y.reshape(shape)
        return (y, stream.reshape(shape)) if prenorm else y

    @staticmethod
    def backward(ctx, dy, *d_stream):
        stream, weight, bias, mean, rstd = ctx.saved_tensors
        shape, x_dtype, is_rms, had_residual, prenorm = ctx.meta
        dy2 = _rows(dy)
        if dy2.shape != stream.shape:
            raise RuntimeError("layer_norm_fn backward: gradient shape does not match the forward's rows")
        g_stream = None
        if prenorm:                      # gradient arriving through the returned residual stream
            g_stream = _rows(d_stream[0])
            if g_stream.dtype != stream.dtype:
                g_stream = g_stream.to(stream.dtype)
        dx, dw, db, d_res = _norm_bwd(dy2, stream, weight, bias, mean, rstd, g_stream, had_residual, is_rms, x_dtype)
        return (dx.reshape(shape), dw, db, d_res.reshape(shape) if had_residual else None, None, None, None, None)


def layer_norm_fn(x, weight, bias, residual=None, eps=1e-6, prenorm=False, residual_in_fp32=False,
                  is_rms_norm=False):
    return LayerNormFn.apply(x, weight, bias, residual, eps, prenorm, residual_in_fp32, is_rms_norm)


def rms_norm_fn(x, weight, bias, residual=None, prenorm=False, residual_in_fp32=False, eps=1e-6):
    return LayerNormFn.apply(x, weight, bias, residual, eps, prenorm, residual_in_fp32, True)


class RMSNorm(torch.nn.Module):
    """Module form of ``rms_norm_fn``.  State-dict contract of the reference's class (layernorm.py:481-503): one parameter
    ``weight`` of size hidden_size (ones at init), ``bias`` registered as None, ``eps`` an attribute."""

    def __init__(self, hidden_size, eps=1e-5, device=None, dtype=None):
        super().__init__()
        self.eps = eps
        self.weight = torch.nn.Parameter(torch.ones(hidden_size, device=device, dtype=dtype))
        self.register_parameter("bias", None)

    def reset_parameters(self):
        with torch.no_grad():
            self.weight.fill_(1.0)

    def forward(self, x, residual=None, prenorm=False, residual_in_fp32=False):
        return LayerNormFn.apply(x, self.weight, None, residual, self.eps, prenorm, residual_in_fp32, True)
