"""bf16 GEMM on the Hopper tensor cores (wgmma): ``linear_bf16(x, weight, bias)`` == ``F.linear`` for row-major
bf16 activations and an ``nn.Linear`` weight (N, K) -- the dense projections of the hot path
(mamba_simple.py:290-294, selective_scan_interface.py:322-323,365).  C-ABI: zg_gemm_bf16_tn."""
import torch

from . import _lib


def linear_bf16(x, weight, bias=None, out=None, out_rowmap=None, rows_per_batch=0):
    """x: (M, K) bf16 with unit inner stride; weight: (N, K) bf16; returns (M, N) bf16.
    out_rowmap (int32[rows_per_batch]): output row m of batch m // rows_per_batch is written to row
    out_rowmap[m % rows_per_batch] of that batch (fused scatter of the out_proj result)."""
    _lib.require_cuda(x, weight, bias)
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
    if out is None:
        out = torch.empty((M, N), dtype=torch.bfloat16, device=x.device)
    p = _lib.GemmParams()
    p.A, p.B, p.bias, p.C = _lib.ptr(x), _lib.ptr(weight), _lib.ptr(bias.contiguous() if bias is not None else None), _lib.ptr(out)
    p.out_rowmap = _lib.ptr(out_rowmap)
    p.lda, p.ldb, p.ldc = x.stride(0), weight.stride(0), out.stride(0)
    p.M, p.N, p.K, p.rows_per_batch = M, N, K, rows_per_batch
    _lib.call("zg_gemm_bf16_tn", p)
    return out
