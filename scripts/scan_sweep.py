"""Times the selective-scan forward kernel at a layer shape (default BASELINE config 2: bs=64, E=1280, L=1024, N=16, bf16,
token-major, z through the zigzag table).  The kernel choice is made by environment variables read once per process
(ZG_SCAN_TMA, ZG_SCAN_PLAIN; ZG_SCAN_WP / ZG_SCAN_WPH_ND / ZG_SCAN_WPH_NS are read per call): run once per setting.  FUSED=1 times the fused dt_proj prologue
(no delta tensor) next to the two-kernel route dt_proj GEMM + scan."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from zigma_b200.selective_scan_interface import _scan_fwd
from zigma_b200 import zigzag_path
from zigma_b200.engine import _linear
dev = "cuda"
bs, L, E, N = [int(os.environ.get(k, v)) for k, v in (("BS", 64), ("SEQ", 1024), ("EDIM", 1280), ("NST", 16))]
R = E // 2 // 16
gen = torch.Generator(device=dev).manual_seed(0)
dt = torch.bfloat16
xz = torch.randn(bs, L, 2 * E, device=dev, generator=gen).to(dt)
xc = torch.randn(bs, L, E, device=dev, generator=gen).to(dt)
xdbl = torch.randn(bs, L, R + 2 * N, device=dev, generator=gen).to(dt)
wdt = (torch.randn(E, R, device=dev, generator=gen) * R ** -0.5).to(dt)
A = -0.5 * torch.rand(E, N, device=dev, generator=gen) - 0.05
Dp, bias = torch.randn(E, device=dev, generator=gen), 0.5 * torch.rand(E, device=dev, generator=gen) - 3.0
side = int(round(L ** 0.5))
perm = torch.from_numpy(zigzag_path(side)[1]).to(dev).to(torch.int32) if side * side == L else torch.randperm(L, device=dev).to(torch.int32)
Bv = xdbl[:, :, R:R + N].permute(0, 2, 1).unsqueeze(1)
Cv = xdbl[:, :, R + N:].permute(0, 2, 1).unsqueeze(1)
outb = torch.empty(bs, L, E, device=dev, dtype=dt).transpose(1, 2)
outf = torch.empty(bs, L, E, device=dev, dtype=dt).transpose(1, 2)
z_log = xz[:, :, E:].transpose(1, 2)
gemm = lambda: _linear(xdbl.view(bs * L, -1)[:, :R], wdt)
dl = gemm().view(bs, L, E)
tok = lambda: _scan_fwd(xc.transpose(1, 2), dl.transpose(1, 2), A, Bv, Cv, Dp, z_log, bias, True, z_rowmap=perm, want_last_state=False, out=outb)
fused = lambda: _scan_fwd(xc.transpose(1, 2), None, A, Bv, Cv, Dp, z_log, bias, True, z_rowmap=perm, want_last_state=False, out=outf, dt_proj=(wdt, xdbl))
def timeit(fn, n=20):
    for _ in range(3): fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(n): fn()
    b.record(); torch.cuda.synchronize()
    return a.elapsed_time(b) / n
t_tok = timeit(tok)
abytes = 4 * 2 * bs * E * L + 2 * 2 * bs * N * L + 4 * (E * N + 2 * E)
tag = " ".join(f"{k}={os.environ[k]}" for k in ("ZG_SCAN_TMA", "ZG_SCAN_PLAIN", "ZG_SCAN_WP", "ZG_SCAN_WPH_ND", "ZG_SCAN_WPH_NS", "ZIGMA_B200_LIB") if k in os.environ) or "default"
line = f"[{tag}] bs={bs} L={L} E={E}: scan {t_tok:.4f} ms ({abytes / t_tok / 1e6:.0f} GB/s of {abytes / 1e6:.0f} MB)"
if os.environ.get("FUSED", "1") == "1" and R in (40, 48) and L % 8 == 0:
    t_gemm, t_fused = timeit(gemm), timeit(fused)
    tok(); fused(); torch.cuda.synchronize()
    diff = (outb.float() - outf.float()).abs().max().item()
    nbad = (outb != outf).float().mean().item()
    line += f" | dt_proj GEMM {t_gemm:.4f} ms, fused scan {t_fused:.4f} ms (vs {t_tok + t_gemm:.4f}); fused vs 2-kernel max|diff| {diff:.3e}, differing elements {nbad:.2e}"
print(line)
