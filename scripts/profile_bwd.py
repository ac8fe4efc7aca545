"""One launch of every TRAINING kernel at the BASELINE config-2 layer shape (token-major, bf16), to run under a profiler."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from zigma_b200.selective_scan_interface import _scan_fwd, _scan_bwd
from zigma_b200.causal_conv1d_interface import _conv_bwd
from zigma_b200 import rms_norm_fn, zigzag_path
dev = "cuda"
bs, L, E, D, N = int(os.environ.get("BS", 16)), 1024, 1280, 640, 16
dt = torch.bfloat16
g = torch.Generator(device=dev).manual_seed(0)
tm = lambda a: a.transpose(-1, -2).contiguous().transpose(-1, -2)
u = tm(torch.randn(bs, E, L, device=dev, generator=g).to(dt)); z = tm(torch.randn(bs, E, L, device=dev, generator=g).to(dt))
delta = tm((0.5 * torch.rand(bs, E, L, device=dev, generator=g)).to(dt))
B = tm(torch.randn(bs, 1, N, L, device=dev, generator=g).to(dt)); C = tm(torch.randn(bs, 1, N, L, device=dev, generator=g).to(dt))
A = -0.5 * torch.rand(E, N, device=dev, generator=g); Dp = torch.randn(E, device=dev, generator=g); bias = 0.5 * torch.rand(E, device=dev, generator=g)
dout = tm(torch.randn(bs, E, L, device=dev, generator=g).to(dt))
perm = torch.from_numpy(zigzag_path(32)[1]).to(dev).to(torch.int32)
w = torch.randn(E, 4, device=dev, generator=g).to(dt); cb = torch.randn(E, device=dev, generator=g).to(dt)
x = torch.randn(bs * L, D, device=dev, generator=g).to(dt).requires_grad_(); res = torch.randn(bs * L, D, device=dev, generator=g).requires_grad_()
nw = torch.ones(D, device=dev, dtype=dt).requires_grad_()
for it in range(2):
    torch.cuda.synchronize()
    if it == 1: torch.cuda.profiler.start()
    out, _, ckpt, saved = _scan_fwd(u, delta, A, B, C, Dp, z, bias, True, z_rowmap=perm, want_last_state=False, want_ckpt=True)
    _scan_bwd(saved, ckpt, dout, True, z_rowmap=perm)
    _conv_bwd(u, w, cb, dout, True, x_rowmap=perm)
    y, r = rms_norm_fn(x, nw, None, residual=res, prenorm=True, residual_in_fp32=True, eps=1e-5)
    (y.float().sum() + r.sum()).backward()
    torch.cuda.synchronize()
    if it == 1: torch.cuda.profiler.stop()
