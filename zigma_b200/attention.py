"""Text cross-attention of has_text blocks on the sm_90a kernels (CrossAttention, model_zigma.py:95-135):

    O = softmax(Q K^T / 8) V       per (batch, head), head dimension 64, 1 <= Lk <= 256 text tokens, no mask / dropout

Forward: ``zg_cross_attn_fwd`` (tensor cores for 16-bit, CUDA cores for fp32) reads Q, K, V and writes O token-major, so
the (B, H, L, 64) reshapes and the transpose-and-copy of the library path are not needed.  Backward: ``zg_cross_attn_bwd``
(P recomputed from the saved log-sum-exp; dK / dV summed per segment of query rows into a workspace and added in segment
order, no atomics), so the gradients are bitwise reproducible whether or not ``torch.use_deterministic_algorithms`` is on
(DESIGN.md section 4.7).
"""
import torch

from . import _lib

HEAD_DIM = 64
MAX_KEYS = 256


def _fill_fwd(p, q, k, v, o, lse, heads):
    B, L, dim = q.shape
    p.q, p.k, p.v, p.o, p.lse = q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(), _lib.ptr(lse)
    p.q_sb, p.q_rs, p.k_sb, p.k_rs = q.stride(0), q.stride(1), k.stride(0), k.stride(1)
    p.v_sb, p.v_rs, p.o_sb, p.o_rs = v.stride(0), v.stride(1), o.stride(0), o.stride(1)
    p.batch, p.L, p.Lk, p.heads, p.dim, p.dtype = B, L, k.shape[1], heads, dim, _lib.dt(q)


def _inner_contig(t):
    return t if t.stride(-1) == 1 else t.contiguous()


class CrossAttentionFn(torch.autograd.Function):
    """(q (B, L, H*64), k, v (B, Lk, H*64), heads) -> o (B, L, H*64).  q, k, v may be column slices of one buffer (any
    batch / row strides that keep 16-byte alignment); o and the gradients are contiguous."""

    @staticmethod
    def forward(ctx, q, k, v, heads):
        o, lse = _forward(q, k, v, heads, want_lse=True)
        ctx.save_for_backward(q, k, v, o, lse)
        ctx.heads = heads
        return o

    @staticmethod
    def backward(ctx, do):
        q, k, v, o, lse = ctx.saved_tensors
        do = _inner_contig(do)
        dq, dk, dv = torch.empty_like(o), torch.empty(k.shape, dtype=k.dtype, device=k.device), torch.empty(v.shape, dtype=v.dtype, device=v.device)
        p = _lib.XattnBwdParams()
        _fill_fwd(p.fwd, q, k, v, o, lse, ctx.heads)
        p.dout, p.dq, p.dk, p.dv = do.data_ptr(), dq.data_ptr(), dk.data_ptr(), dv.data_ptr()
        p.dout_sb, p.dout_rs, p.dq_sb, p.dq_rs = do.stride(0), do.stride(1), dq.stride(0), dq.stride(1)
        p.dk_sb, p.dk_rs, p.dv_sb, p.dv_rs = dk.stride(0), dk.stride(1), dv.stride(0), dv.stride(1)
        p.sms = torch.cuda.get_device_properties(q.device).multi_processor_count
        l = _lib.lib()
        nbytes = int(l.zg_cross_attn_bwd_workspace_bytes(_lib.C.byref(p)))
        ws = torch.empty((nbytes,), dtype=torch.uint8, device=q.device)     # torch's allocator, current stream: graph-safe
        stream = torch.cuda.current_stream(q.device).cuda_stream
        rc = l.zg_cross_attn_bwd(_lib.C.byref(p), _lib.C.c_void_p(ws.data_ptr() if nbytes else None), _lib.C.c_int64(nbytes),
                                 _lib.C.c_void_p(stream))
        if rc != 0:
            raise RuntimeError(f"zg_cross_attn_bwd: {l.zg_last_error().decode()}")
        return dq, dk, dv, None


def _forward(q, k, v, heads, want_lse):
    _lib.require_cuda(q, k, v)
    if q.dim() != 3 or k.dim() != 3 or v.dim() != 3:
        raise RuntimeError("cross_attention_fn: q, k, v must be (batch, tokens, heads * 64)")
    if not (q.dtype == k.dtype == v.dtype):
        raise RuntimeError(f"cross_attention_fn: q, k, v dtypes differ ({q.dtype}, {k.dtype}, {v.dtype})")
    if k.shape != v.shape or k.shape[0] != q.shape[0] or k.shape[2] != q.shape[2]:
        raise RuntimeError(f"cross_attention_fn: shapes q {tuple(q.shape)}, k {tuple(k.shape)}, v {tuple(v.shape)} do not match")
    q, k, v = _inner_contig(q), _inner_contig(k), _inner_contig(v)
    B, L, dim = q.shape
    o = torch.empty((B, L, dim), dtype=q.dtype, device=q.device)
    lse = torch.empty((B, heads, L), dtype=torch.float32, device=q.device) if want_lse else None
    p = _lib.XattnParams()
    _fill_fwd(p, q, k, v, o, lse, heads)
    _lib.call("zg_cross_attn_fwd", p)
    return o, lse


def cross_attention_fn(q, k, v, heads):
    """softmax(q k^T / 8) v per head on the sm_90a kernels: q (B, L, heads * 64), k / v (B, Lk, heads * 64) with
    1 <= Lk <= 256, one dtype (fp32, fp16 or bf16), innermost dimension contiguous.  Differentiable; the log-sum-exp the
    backward needs is written only when a gradient is required."""
    if torch.is_grad_enabled() and any(t.requires_grad for t in (q, k, v)):
        return CrossAttentionFn.apply(q, k, v, heads)
    return _forward(q, k, v, heads, want_lse=False)[0]
