"""bf16 GEMM on the Hopper tensor cores (wgmma): ``linear_bf16(x, weight, bias)`` == ``F.linear`` for row-major
bf16 activations and an ``nn.Linear`` weight (N, K) -- the dense projections of the hot path
(mamba_simple.py:290-294, selective_scan_interface.py:322-323,365).  C-ABI: zg_gemm_bf16_tn."""
import torch

from . import _lib


def linear_bf16(x, weight, bias=None, out=None, out_rowmap=None, rows_per_batch=0):
    """x: (M, K) bf16 with unit inner stride; weight: (N, K) bf16; bias: contiguous bf16 (N,); returns (M, N) bf16, written
    into ``out`` when given (bf16, shape (M, N), unit column stride, any row stride that is at least N).
    out_rowmap (contiguous int32[rows_per_batch], rows_per_batch dividing M): output row m of batch m // rows_per_batch is
    written to row out_rowmap[m % rows_per_batch] of that batch (fused scatter of the out_proj result).  Its values are not
    checked (that would need a device sync): they must lie in [0, rows_per_batch), or the kernel writes outside ``out``."""
    _lib.require_cuda(x, weight, bias, out, out_rowmap)
    if x.dtype != torch.bfloat16 or weight.dtype != torch.bfloat16:
        raise RuntimeError("linear_bf16: bf16 operands required")
    if x.dim() != 2 or weight.dim() != 2 or x.shape[1] != weight.shape[1]:
        raise RuntimeError("linear_bf16: shapes must be (M, K) and (N, K)")
    if x.stride(1) != 1:
        x = x.contiguous()
    if weight.stride(1) != 1:
        weight = weight.contiguous()
    if x.stride(0) % 8 or weight.stride(0) % 8:
        raise RuntimeError("linear_bf16: leading dimensions must be multiples of 8 elements (16-byte TMA pitch)")
    M, K = x.shape
    N = weight.shape[0]
    for name, t in (("weight", weight), ("bias", bias), ("out", out), ("out_rowmap", out_rowmap)):
        if t is not None and t.device != x.device:
            raise RuntimeError(f"linear_bf16: {name} is on {t.device}, x on {x.device}")
    if bias is not None and (bias.dtype != torch.bfloat16 or bias.numel() != N or not bias.is_contiguous()):
        raise RuntimeError(f"linear_bf16: bias must be a contiguous bf16 tensor of N = {N} elements, got {bias.dtype} "
                           f"{tuple(bias.shape)} with strides {bias.stride()}")
    if out is None:
        out = torch.empty((M, N), dtype=torch.bfloat16, device=x.device)
    elif out.dtype != torch.bfloat16 or tuple(out.shape) != (M, N) or out.stride(1) != 1:
        raise RuntimeError(f"linear_bf16: out must be bf16 of shape ({M}, {N}) with unit column stride, got {out.dtype} "
                           f"{tuple(out.shape)} with strides {out.stride()}")
    if out_rowmap is not None and (out_rowmap.dtype != torch.int32 or out_rowmap.numel() != rows_per_batch
                                   or not out_rowmap.is_contiguous()):
        raise RuntimeError(f"linear_bf16: out_rowmap must be a contiguous int32 tensor of rows_per_batch = {rows_per_batch} "
                           f"elements, got {out_rowmap.dtype} {tuple(out_rowmap.shape)} with strides {out_rowmap.stride()}")
    p = _lib.GemmParams()
    p.A, p.B, p.bias, p.C = _lib.ptr(x), _lib.ptr(weight), _lib.ptr(bias), _lib.ptr(out)
    p.out_rowmap = _lib.ptr(out_rowmap)
    p.lda, p.ldb, p.ldc = x.stride(0), weight.stride(0), out.stride(0)
    p.M, p.N, p.K, p.rows_per_batch = M, N, K, rows_per_batch
    _lib.call("zg_gemm_bf16_tn", p)
    return out
