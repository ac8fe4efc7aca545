"""wgmma GEMM (zg_gemm_bf16_tn) vs the library GEMM at the four projection shapes of BASELINE config 2."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch, torch.nn.functional as F
from zigma_b200.gemm import linear_bf16
dev = "cuda"
M = 65536
def timeit(fn, n=20):
    for _ in range(3): fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(n): fn()
    b.record(); torch.cuda.synchronize()
    return a.elapsed_time(b) / n
for name, N, K in (("in_proj", 2560, 640), ("out_proj", 640, 1280), ("x_proj", 72, 1280), ("dt_proj", 1280, 40)):
    Kp = (K + 7) // 8 * 8
    x = torch.randn(M, Kp, device=dev).bfloat16()[:, :K]
    w = (torch.randn(N, Kp, device=dev) / K ** 0.5).bfloat16()[:, :K]
    out = torch.empty(M, N, device=dev, dtype=torch.bfloat16)
    t_ours = timeit(lambda: linear_bf16(x, w, out=out))
    t_lib = timeit(lambda: F.linear(x, w))
    fl = 2.0 * M * N * K
    err = (linear_bf16(x, w).float() - F.linear(x, w).float()).abs().max().item()
    print(f"{name:9s} M={M} N={N} K={K}: wgmma {t_ours*1e3:7.1f} us ({fl/t_ours/1e9:7.1f} TFLOP/s)   library {t_lib*1e3:7.1f} us ({fl/t_lib/1e9:7.1f} TFLOP/s)   max|diff| {err:.3e}")
