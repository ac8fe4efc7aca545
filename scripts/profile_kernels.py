"""One launch of every hot-path kernel at the BASELINE config-2 layer shape, to run under a profiler."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from zigma_b200.selective_scan_interface import _scan_fwd
from zigma_b200.causal_conv1d_interface import _conv_fwd
from zigma_b200.engine import block_tail
from zigma_b200.gemm import linear_bf16
from zigma_b200 import zigzag_path, reverse_permut_np
dev = "cuda"
bs, L, E, D, N, R = 64, 1024, 1280, 640, 16, 40
dt = torch.bfloat16
g = torch.Generator(device=dev).manual_seed(0)
xz = torch.randn(bs, L, 2 * E, device=dev, generator=g).to(dt)
xc = torch.randn(bs, L, E, device=dev, generator=g).to(dt)
dl = (0.5 * torch.rand(bs, L, E, device=dev, generator=g)).to(dt)
xdbl = torch.randn(bs, L, R + 2 * N, device=dev, generator=g).to(dt)
A = -0.5 * torch.rand(E, N, device=dev, generator=g)
Dp, bias = torch.randn(E, device=dev, generator=g), 0.5 * torch.rand(E, device=dev, generator=g)
perm = torch.from_numpy(zigzag_path(32)[1]).to(dev).to(torch.int32)
rev = torch.from_numpy(reverse_permut_np(zigzag_path(32)[1])).to(dev).to(torch.int32)
Bv = xdbl[:, :, R:R + N].permute(0, 2, 1).unsqueeze(1)
Cv = xdbl[:, :, R + N:].permute(0, 2, 1).unsqueeze(1)
w, b = torch.randn(E, 4, device=dev, generator=g).to(dt), torch.randn(E, device=dev, generator=g).to(dt)
x = torch.randn(bs, L, D, device=dev, generator=g).to(dt); mix = torch.randn(bs, L, D, device=dev, generator=g).to(dt)
mods = torch.randn(bs, 3 * D, device=dev, generator=g).to(dt); res = torch.randn(bs, L, D, device=dev, generator=g); nw = torch.ones(D, device=dev).to(dt)
Win = (torch.randn(2 * E, D, device=dev, generator=g) / D ** 0.5).to(dt)
Wout = (torch.randn(D, E, device=dev, generator=g) / E ** 0.5).to(dt)
for it in range(2):     # first pass warms up (attributes, caches); profile the second
    torch.cuda.synchronize()
    if it == 1: torch.cuda.profiler.start()
    _scan_fwd(xc.transpose(1, 2), dl.transpose(1, 2), A, Bv, Cv, Dp, xz[:, :, E:].transpose(1, 2), bias, True, z_rowmap=perm, want_last_state=False)
    _conv_fwd(xz[:, :, :E].transpose(1, 2), w, b, True, x_rowmap=perm)
    block_tail(x, mix, mods[:, :D], mods[:, D:2 * D], mods[:, 2 * D:], nw, res, rev, 1e-5)
    linear_bf16(x.reshape(bs * L, D), Win)
    linear_bf16(xc.reshape(bs * L, E), Wout)
    torch.cuda.synchronize()
    if it == 1: torch.cuda.profiler.stop()
