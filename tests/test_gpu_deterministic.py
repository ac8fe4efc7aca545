"""GPU: torch.use_deterministic_algorithms(True) makes every backward op of the package bitwise reproducible.

Per op and dispatch branch: the deterministic path runs once on an idle device and once while a second stream runs a long
independent matmul (which changes the order in which CTAs run); both results must be bitwise equal, agree with the atomic
(flag off) path to fp32 reordering accuracy and, where golden gradients exist, with those.  The whole-training-step check
runs tests/_det_train_worker.py twice in fresh processes and compares the digests."""
import os
import subprocess
import sys

import pytest
import torch

from util import ROOT, check_close, gold, t

pytestmark = pytest.mark.gpu
DEV = "cuda"


class _Load:
    """A long chain of independent matmuls on a side stream (queued with the flag off: cuBLAS's own determinism rules do
    not concern it), so that the op under test shares the SMs with it."""

    def __enter__(self):
        self.stream = torch.cuda.Stream()
        self.stream.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(self.stream):
            a = torch.randn(4096, 4096, device=DEV)
            for _ in range(24):
                a = torch.tanh(a @ a * 1e-2)
        self.keep = a
        return self

    def __exit__(self, *exc):
        torch.cuda.current_stream().wait_stream(self.stream)
        torch.cuda.synchronize()


def _run(fn, deterministic):
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(deterministic)
    try:
        out = fn()
    finally:
        torch.use_deterministic_algorithms(prev)
    torch.cuda.synchronize()
    return [None if o is None else o.detach().clone() for o in out]


def _check(fn, names, rtol=1e-3, atol=1e-5, golden=None, golden_tol=None):
    """fn() -> tuple of outputs.  Deterministic idle == deterministic under load (bitwise), close to the atomic path: the
    hard bound of util.check_close (absolute floor scaled by the output range -- a column sum over thousands of rows in
    another order moves the small entries by more than their own rtol, so the strict-fraction check does not apply)."""
    det = _run(fn, True)
    with _Load():
        det_loaded = _run(fn, True)
    det_again = _run(fn, True)
    ref = _run(fn, False)
    for n, a, b, c, r in zip(names, det, det_loaded, det_again, ref):
        if a is None:
            continue
        assert torch.equal(a, b), f"{n}: deterministic backward differs under load (max|diff| {(a.float() - b.float()).abs().max().item():.3e})"
        assert torch.equal(a, c), f"{n}: deterministic backward differs between two idle runs"
        check_close(a, r, f"{n} det vs atomic", rtol=rtol, atol=atol, max_strict_viol=1.0)
        if golden is not None and n in golden:
            check_close(a, golden[n], f"{n} det vs golden", **(golden_tol or {}))
    return det


# ---- selective scan ----------------------------------------------------------------------------------------------------
def _scan_case(batch, dim, L, dstate, token_major, dtype, rowmap=False, const_bc=False, seed=0):
    from zigma_b200.selective_scan_interface import _scan_bwd, _scan_fwd
    g = torch.Generator(device=DEV).manual_seed(seed)
    rnd = lambda *s: torch.randn(*s, device=DEV, generator=g)
    act = lambda: (rnd(batch, L, dim).transpose(1, 2) if token_major else rnd(batch, dim, L)).to(dtype)
    u, z, dout = act(), act(), act()
    delta = (0.5 * torch.rand(batch, L, dim, device=DEV, generator=g)).transpose(1, 2) if token_major else 0.5 * torch.rand(batch, dim, L, device=DEV, generator=g)
    delta = delta.to(dtype)
    A = -0.5 * torch.rand(dim, dstate, device=DEV, generator=g)
    if const_bc:
        B, C = rnd(dim, dstate), rnd(dim, dstate)
    elif token_major:
        B, C = [rnd(batch, L, 1, dstate).permute(0, 2, 3, 1).to(dtype) for _ in range(2)]
    else:
        B, C = [rnd(batch, 1, dstate, L).to(dtype) for _ in range(2)]
    D, bias = rnd(dim), 0.5 * torch.rand(dim, device=DEV, generator=g)
    zr = torch.randperm(L, device=DEV, generator=g).to(torch.int32) if rowmap else None
    _, _, ckpt, saved = _scan_fwd(u, delta, A, B, C, D, z, bias, True, z_rowmap=zr, want_last_state=False, want_ckpt=True)
    return lambda: _scan_bwd(saved, ckpt, dout, True, z_rowmap=zr)


SCAN_NAMES = ["du", "ddelta", "dA", "dB", "dC", "dD", "ddelta_bias", "dz"]


@pytest.mark.parametrize("case", ["q4_staged_token_major_rowmap", "q4_staged_channel_first", "q4_unstaged_ragged", "generic_dstate8",
                                  "generic_constant_bc", "q4_staged_bf16_config2_width"])
def test_scan_bwd_deterministic(case):
    fn = {
        "q4_staged_token_major_rowmap": lambda: _scan_case(2, 128, 64, 16, True, torch.bfloat16, rowmap=True),
        "q4_staged_channel_first": lambda: _scan_case(2, 128, 64, 16, False, torch.float32),
        "q4_unstaged_ragged": lambda: _scan_case(2, 96, 45, 16, False, torch.float32),
        "generic_dstate8": lambda: _scan_case(2, 64, 50, 8, False, torch.float32),
        "generic_constant_bc": lambda: _scan_case(2, 64, 50, 16, False, torch.float32, const_bc=True),
        "q4_staged_bf16_config2_width": lambda: _scan_case(4, 1280, 256, 16, True, torch.bfloat16, rowmap=True),
    }[case]()
    _check(fn, SCAN_NAMES)


@pytest.mark.parametrize("name", ["e64_n16", "e96_l45_n16", "n4", "e128_g2_n16"])
def test_scan_bwd_deterministic_golden(name):
    """selective_scan_fn's gradients under the flag against the golden gradients (the tolerances of test_gpu_bwd)."""
    from zigma_b200 import selective_scan_fn
    g = gold("scan_" + name)
    Bt, E, L, N, G, hasD, hasz, hasb, sp = [int(v) for v in g["flags"]]
    names = ["u", "delta", "A", "B", "C"] + (["D"] if hasD else []) + (["z"] if hasz else []) + (["delta_bias"] if hasb else [])

    def fn():
        req = {k: t(g[k], DEV).requires_grad_() for k in ("u", "delta", "A", "B", "C", "D", "z", "delta_bias")}
        Bm = req["B"] if G > 1 else req["B"][:, 0]
        Cm = req["C"] if G > 1 else req["C"][:, 0]
        out = selective_scan_fn(req["u"], req["delta"], req["A"], Bm, Cm, req["D"] if hasD else None, z=req["z"] if hasz else None,
                                delta_bias=req["delta_bias"] if hasb else None, delta_softplus=bool(sp))
        out.backward(t(g["g"], DEV))
        return [req[k].grad for k in names]
    _check(fn, ["d" + k for k in names], golden={"d" + k: g["d" + k] for k in names}, golden_tol=dict(atol=1e-4, max_strict_viol=1e-2))


# ---- causal conv1d -------------------------------------------------------------------------------------------------------
def _conv_case(batch, dim, L, token_major, dtype, rowmap=False, seed=1):
    from zigma_b200.causal_conv1d_interface import _conv_bwd
    g = torch.Generator(device=DEV).manual_seed(seed)
    act = lambda: (torch.randn(batch, L, dim, device=DEV, generator=g).transpose(1, 2) if token_major
                   else torch.randn(batch, dim, L, device=DEV, generator=g)).to(dtype)
    x, dout = act(), act()
    w, b = 0.5 * torch.randn(dim, 4, device=DEV, generator=g), torch.randn(dim, device=DEV, generator=g)
    xr = torch.randperm(L, device=DEV, generator=g).to(torch.int32) if rowmap else None
    return lambda: _conv_bwd(x, w, b, dout, True, x_rowmap=xr)


@pytest.mark.parametrize("case", ["tok4", "tok4_rowmap", "tok_fp32", "tok_unaligned", "seqc", "seqc_vec"])
def test_conv_bwd_deterministic(case):
    fn = {
        "tok4": lambda: _conv_case(3, 256, 128, True, torch.bfloat16),
        "tok4_rowmap": lambda: _conv_case(3, 256, 128, True, torch.bfloat16, rowmap=True),
        "tok_fp32": lambda: _conv_case(3, 96, 150, True, torch.float32),
        "tok_unaligned": lambda: _conv_case(3, 6, 150, True, torch.bfloat16),
        "seqc": lambda: _conv_case(3, 40, 151, False, torch.float32),
        "seqc_vec": lambda: _conv_case(3, 40, 256, False, torch.bfloat16),
    }[case]()
    _check(fn, ["dx", "dweight", "dbias"])


def test_conv_bwd_deterministic_golden():
    from zigma_b200 import causal_conv1d_fn
    g = gold("conv")

    def fn():
        x, w, b = t(g["x"], DEV).requires_grad_(), t(g["w4"], DEV).requires_grad_(), t(g["b4"], DEV).requires_grad_()
        causal_conv1d_fn(x, w, b, activation="silu").backward(t(g["g"], DEV))
        return x.grad, w.grad, b.grad
    _check(fn, ["dx", "dw", "db"], golden={"dx": g["dx_W4_s1_b1"], "dw": g["dw_W4_s1_b1"], "db": g["db_W4_s1_b1"]})


# ---- fused add + norm ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", ["vec_rms", "vec_layernorm", "plain_wide"])
def test_add_norm_bwd_deterministic(case):
    """Against the atomic path and against autograd through the eager formula in fp64."""
    from zigma_b200.layernorm import layer_norm_fn, rms_norm_fn
    ncols = {"vec_rms": 640, "vec_layernorm": 640, "plain_wide": 1280}[case]
    rms = case != "vec_layernorm"
    g = torch.Generator(device=DEV).manual_seed(2)
    x0, r0, dy = [torch.randn(4000, ncols, device=DEV, generator=g) for _ in range(3)]
    w0, b0 = 1 + 0.1 * torch.randn(ncols, device=DEV, generator=g), 0.1 * torch.randn(ncols, device=DEV, generator=g)

    def fn():
        x, r, w = x0.clone().requires_grad_(), r0.clone().requires_grad_(), w0.clone().requires_grad_()
        b = None if rms else b0.clone().requires_grad_()
        y = (rms_norm_fn(x, w, None, residual=r, eps=1e-5) if rms else layer_norm_fn(x, w, b, residual=r, eps=1e-5))
        y.backward(dy)
        return x.grad, r.grad, w.grad, (None if rms else b.grad)
    got = _check(fn, ["dx", "dres", "dw", "db"])
    x, r, w = x0.double().requires_grad_(), r0.double(), w0.double().requires_grad_()
    b = None if rms else b0.double().requires_grad_()
    h = x + r
    y = (h * torch.rsqrt(h.square().mean(-1, keepdim=True) + 1e-5) * w if rms
         else torch.nn.functional.layer_norm(h, (ncols,), w, b, eps=1e-5))
    y.backward(dy.double())
    check_close(got[0], x.grad, "dx vs fp64")
    check_close(got[2], w.grad, "dw vs fp64", atol=1e-4)
    if not rms:
        check_close(got[3], b.grad, "db vs fp64", atol=1e-4)


# ---- block tail ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", ["rowmap", "no_mix", "ragged_batches"])
def test_block_tail_bwd_deterministic(case):
    from zigma_b200.block_ops import block_tail_fn
    B, L, D = {"rowmap": (4, 256, 640), "no_mix": (4, 256, 640), "ragged_batches": (3, 37, 128)}[case]
    dtype = torch.bfloat16
    g = torch.Generator(device=DEV).manual_seed(3)
    rnd = lambda *s: torch.randn(*s, device=DEV, generator=g)
    x0, mix0 = rnd(B, L, D).to(dtype), rnd(B, L, D).to(dtype)
    ada = (0.5 * rnd(B, 3 * D)).to(dtype)
    res0, nw0 = rnd(B, L, D), (1 + 0.1 * rnd(D)).to(dtype)
    rowmap = torch.randperm(L, device=DEV, generator=g).to(torch.int32) if case != "no_mix" else None
    gr, gn, gm = rnd(B, L, D), rnd(B, L, D).to(dtype), rnd(B, L, D).to(dtype)
    first = case == "no_mix"

    def fn():
        x, nw = x0.clone().requires_grad_(), nw0.clone().requires_grad_()
        a = ada.clone().requires_grad_()
        gate, shift, scale = a.chunk(3, dim=1)
        mix = None if first else mix0.clone().requires_grad_()
        res = None if first else res0.clone().requires_grad_()
        out = block_tail_fn(x, mix, None if first else gate, shift, scale, nw, res, rowmap, 1e-5)
        torch.autograd.backward(out, (gr, gn, gm))
        return x.grad, a.grad, nw.grad, (None if first else mix.grad), (None if first else res.grad)
    got = _check(fn, ["dx", "d_ada", "d_norm_w", "d_mix", "d_residual"], rtol=2e-2, atol=2e-2)
    # the eager composition in fp32 (the bf16 rounding points of the kernel are those of the unfused graph)
    x = x0.float().requires_grad_()
    a = ada.float().requires_grad_()
    gate, shift, scale = a.chunk(3, dim=1)
    nw = nw0.float().requires_grad_()
    hidden = x if first else x + gate[:, None] * mix0.float()[:, rowmap.long()]
    rr = hidden if first else res0 + hidden
    normed = rr * torch.rsqrt(rr.square().mean(-1, keepdim=True) + 1e-5) * nw
    modded = normed * (1 + scale[:, None]) + shift[:, None]
    torch.autograd.backward((rr, normed, modded), (gr, gn.float(), gm.float()))
    check_close(got[1].float(), a.grad, "d_ada vs fp32 eager", rtol=3e-2, atol=3e-2, max_strict_viol=1.0)
    check_close(got[2].float(), nw.grad, "d_norm_w vs fp32 eager", rtol=3e-2, atol=3e-2, max_strict_viol=1.0)


# ---- whole training steps -------------------------------------------------------------------------------------------------
def test_train_steps_are_bitwise_reproducible():
    """Two fresh processes, same seeds: identical digests of parameters, Adam moments, EMA, losses and bf16 gradients for every
    supported configuration, and no error from PyTorch's own deterministic checks."""
    worker = os.path.join(ROOT, "tests", "_det_train_worker.py")
    runs = []
    for _ in range(2):
        r = subprocess.run([sys.executable, worker], capture_output=True, text=True, timeout=1800, cwd=ROOT)
        assert r.returncode == 0 and "DET_WORKER_OK" in r.stdout, r.stdout[-3000:] + r.stderr[-6000:]
        runs.append([l for l in r.stdout.splitlines() if l.startswith("DIGEST ")])
    assert len(runs[0]) > 50
    diff = [(a, b) for a, b in zip(*runs) if a != b]
    assert len(runs[0]) == len(runs[1]) and not diff, diff[:10]
