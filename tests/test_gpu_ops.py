"""GPU (H100): parity of every op of the C-ABI against the oracle / the reference's golden vectors.
All calls go through the host mirror of the reference interface -> ctypes -> libzigma_b200.so."""
import numpy as np
import pytest
import torch

from oracle import c_oracle, synth, zigma_oracle as zo
from util import check_close, gold, t

pytestmark = pytest.mark.gpu
DEV = "cuda"

SCAN = ["t128_g1", "t131_g2", "e64_n16", "plain", "noz", "l1", "l16_many", "n4", "e128_g2_n16", "e96_l45_n16"]


def _scan_args(g, dev=DEV, dtype=None):
    Bt, E, L, N, G, hasD, hasz, hasb, sp = [int(v) for v in g["flags"]]
    c = lambda k: t(g[k], dev, dtype)
    B, C = c("B"), c("C")
    return dict(u=c("u"), delta=c("delta"), A=t(g["A"], dev), B=B if G > 1 else B[:, 0], C=C if G > 1 else C[:, 0],
                D=t(g["D"], dev) if hasD else None, z=c("z") if hasz else None,
                delta_bias=t(g["delta_bias"], dev) if hasb else None, delta_softplus=bool(sp)), (Bt, E, L, N, G)


@pytest.mark.parametrize("name", SCAN)
def test_selective_scan_fwd_golden_fp32(name):
    """selective_scan_fn in the reference (channel-first) layout vs the reference's own output."""
    from zigma_b200 import selective_scan_fn
    g = gold("scan_" + name)
    a, _ = _scan_args(g)
    out, last = selective_scan_fn(a["u"], a["delta"], a["A"], a["B"], a["C"], a["D"], z=a["z"], delta_bias=a["delta_bias"],
                                  delta_softplus=a["delta_softplus"], return_last_state=True)
    check_close(out, g["out"], f"scan {name} out")
    check_close(last, g["last_state"], f"scan {name} last_state")


@pytest.mark.parametrize("name", SCAN)
def test_selective_scan_fwd_token_major_golden_fp32(name):
    """Same vectors through the dim-contiguous (token-major) loader: u, delta, z as transposed views
    of (B, L, E) tensors, B/C as (B, G, N, L) views of (B, G, L, N) memory."""
    from zigma_b200 import selective_scan_fn
    g = gold("scan_" + name)
    a, (Bt, E, L, N, G) = _scan_args(g)
    tm = lambda x: None if x is None else x.transpose(1, 2).contiguous().transpose(1, 2)
    Bv = a["B"] if a["B"].dim() == 4 else a["B"].unsqueeze(1)
    Cv = a["C"] if a["C"].dim() == 4 else a["C"].unsqueeze(1)
    Bv = Bv.transpose(2, 3).contiguous().transpose(2, 3)
    Cv = Cv.transpose(2, 3).contiguous().transpose(2, 3)
    out, last = selective_scan_fn(tm(a["u"]), tm(a["delta"]), a["A"], Bv, Cv, a["D"], z=tm(a["z"]), delta_bias=a["delta_bias"],
                                  delta_softplus=a["delta_softplus"], return_last_state=True)
    assert out.shape == (Bt, E, L)
    check_close(out, g["out"], f"scan(token-major) {name} out")
    check_close(last, g["last_state"], f"scan(token-major) {name} last_state")


def test_selective_scan_config1_fp32():
    """BASELINE config 1: B=2 L=1024 D=640 N=16 fp32, against the reference digest and the C oracle."""
    from zigma_b200 import selective_scan_fn
    g = gold("scan_config1_digest")
    inp = synth.synth_scan_inputs(2, 640, 1024, 16, 1, seed=2)
    d = {k: v.to(DEV) for k, v in inp.items()}
    out, last = selective_scan_fn(d["u"], d["delta"], d["A"], d["B"], d["C"], d["D"], z=d["z"], delta_bias=d["delta_bias"],
                                  delta_softplus=True, return_last_state=True)
    o = out.cpu()
    check_close(o.reshape(-1)[t(g["idx"])], g["out_sub"], "config1 vs reference digest", max_strict_viol=1e-3)
    check_close(last.cpu().reshape(-1)[::13], g["last_sub"], "config1 last_state vs reference digest", max_strict_viol=1e-3)
    ref, ref_last = c_oracle.scan_fwd(inp["u"], inp["delta"], inp["A"], inp["B"], inp["C"], inp["D"], inp["z"], inp["delta_bias"], True)
    check_close(o, ref, "config1 vs C oracle (all 1.3M elements)")
    assert abs(o.double().sum().item() - float(g["out_sum"])) <= 1e-4 * float(g["out_abs_sum"])


@pytest.mark.parametrize("dtype,rtol,atol", [(torch.bfloat16, 1.6e-2, 1e-5), (torch.float16, 2e-3, 1e-5)])
@pytest.mark.parametrize("layout", ["seq", "tok"])
def test_selective_scan_lowp(dtype, rtol, atol, layout):
    """16-bit I/O: inputs rounded to the I/O dtype first, oracle run in fp32 on the rounded inputs,
    result must be the correctly rounded oracle value to within 2 ulp (bf16 ulp = 2^-8, fp16 2^-11)
    (SURVEY.md section 8c protocol item 3)."""
    from zigma_b200 import selective_scan_fn
    Bt, E, L, N = 3, 160, 277, 16
    inp = synth.synth_scan_inputs(Bt, E, L, N, 1, seed=7)
    lo = {k: (v.to(dtype) if k in ("u", "delta", "z", "B", "C") else v) for k, v in inp.items()}
    f32 = {k: v.float().numpy() for k, v in lo.items()}
    ref, ref_last = c_oracle.scan_fwd(f32["u"], f32["delta"], f32["A"], f32["B"], f32["C"], f32["D"], f32["z"], f32["delta_bias"], True)
    d = {k: v.to(DEV) for k, v in lo.items()}
    if layout == "tok":
        tm = lambda x: x.transpose(1, 2).contiguous().transpose(1, 2)
        d["u"], d["delta"], d["z"] = tm(d["u"]), tm(d["delta"]), tm(d["z"])
        d["B"] = d["B"].transpose(2, 3).contiguous().transpose(2, 3)
        d["C"] = d["C"].transpose(2, 3).contiguous().transpose(2, 3)
    out, last = selective_scan_fn(d["u"], d["delta"], d["A"], d["B"], d["C"], d["D"], z=d["z"], delta_bias=d["delta_bias"],
                                  delta_softplus=True, return_last_state=True)
    assert out.dtype == dtype
    check_close(out, ref, f"scan {dtype} {layout}", rtol=rtol, atol=atol, max_strict_viol=1.0)
    check_close(last, ref_last, f"scan {dtype} {layout} last_state (fp32)", max_strict_viol=1e-3)


def test_selective_scan_strided_and_constant_bc():
    """Non-contiguous batch/dim strides (delta as a view of an (E, B*L) GEMM output, u sliced out of a
    wider tensor -- selective_scan_interface.py:323, test_causal_conv1d.py:39-46) and constant B/C."""
    from zigma_b200 import selective_scan_fn
    Bt, E, L, N = 2, 24, 96, 8
    inp = synth.synth_scan_inputs(Bt, E, L, N, 1, seed=9)
    wide = torch.randn(Bt, E + 16, L)
    wide[:, 8:8 + E] = inp["u"]
    u = wide.to(DEV)[:, 8:8 + E]
    delta_el = inp["delta"].permute(1, 0, 2).reshape(E, Bt * L).contiguous().to(DEV)
    delta = delta_el.reshape(E, Bt, L).transpose(0, 1)
    d = {k: v.to(DEV) for k, v in inp.items()}
    out = selective_scan_fn(u, delta, d["A"], d["B"], d["C"], d["D"], z=d["z"], delta_bias=d["delta_bias"], delta_softplus=True)
    ref, _ = c_oracle.scan_fwd(inp["u"], inp["delta"], inp["A"], inp["B"], inp["C"], inp["D"], inp["z"], inp["delta_bias"], True)
    check_close(out, ref, "scan strided views")
    Bc, Cc = torch.randn(E, N), torch.randn(E, N)
    for Bx, Cx, tag in ((Bc, inp["C"][:, 0], "constB"), (inp["B"][:, 0], Cc, "constC"), (Bc, Cc, "constBC")):
        want = zo.selective_scan(inp["u"], inp["delta"], inp["A"], Bx, Cx, inp["D"], inp["z"], inp["delta_bias"], True)
        got = selective_scan_fn(d["u"], d["delta"], d["A"], Bx.to(DEV), Cx.to(DEV), d["D"], z=d["z"], delta_bias=d["delta_bias"], delta_softplus=True)
        check_close(got, want, "scan " + tag)


def test_selective_scan_z_rowmap_fuses_permutation():
    """z_rowmap == gathering z through the zigzag table first (forward_permutation, mamba_simple.py:55-56)."""
    from zigma_b200.selective_scan_interface import _scan_fwd
    import zigma_b200
    Bt, E, L, N = 2, 96, 64, 16
    inp = synth.synth_scan_inputs(Bt, E, L, N, 1, seed=11)
    perm = torch.from_numpy(zigma_b200.zigzag_path(8)[3])
    d = {k: v.to(DEV) for k, v in inp.items()}
    tm = lambda x: x.transpose(1, 2).contiguous().transpose(1, 2)
    Bv = d["B"].transpose(2, 3).contiguous().transpose(2, 3)
    Cv = d["C"].transpose(2, 3).contiguous().transpose(2, 3)
    out, _, _, _ = _scan_fwd(tm(d["u"]), tm(d["delta"]), d["A"], Bv, Cv, d["D"], tm(d["z"]), d["delta_bias"], True,
                             z_rowmap=perm.to(DEV).to(torch.int32), want_last_state=False)
    ref, _ = c_oracle.scan_fwd(inp["u"], inp["delta"], inp["A"], inp["B"], inp["C"], inp["D"], inp["z"][:, :, perm], inp["delta_bias"], True)
    check_close(out, ref, "scan z_rowmap")


def _tok_inputs(Bt, E, L, N, seed, dtype):
    """Token-major 16-bit scan inputs (rounded first) + their fp32 numpy copies for the C oracle."""
    inp = synth.synth_scan_inputs(Bt, E, L, N, 1, seed=seed)
    lo = {k: (v.to(dtype) if k in ("u", "delta", "z", "B", "C") else v) for k, v in inp.items()}
    f32 = {k: v.float().numpy() for k, v in lo.items()}
    d = {k: v.to(DEV) for k, v in lo.items()}
    tm = lambda x: x.transpose(1, 2).contiguous().transpose(1, 2)
    d["u"], d["delta"], d["z"] = tm(d["u"]), tm(d["delta"]), tm(d["z"])
    d["B"] = d["B"].transpose(2, 3).contiguous().transpose(2, 3)
    d["C"] = d["C"].transpose(2, 3).contiguous().transpose(2, 3)
    return d, f32


@pytest.mark.parametrize("dtype,rtol", [(torch.bfloat16, 1.6e-2), (torch.float16, 2e-3)])
@pytest.mark.parametrize("shape", [(2, 192, 264), (3, 64, 8), (1, 128, 1024)])
def test_selective_scan_tma_pipeline_kernel(dtype, rtol, shape):
    """Shapes of the round-2 hot-path kernel (scan_fwd_tma.cuh: token-major, N = 16, L % 8 == 0, E % 64 == 0, 16-bit):
    bulk-async staging + three-phase stages; with the zigzag z_rowmap, the last state and the backward's checkpoints."""
    from zigma_b200.selective_scan_interface import _scan_fwd
    Bt, E, L = shape
    N = 16
    d, f32 = _tok_inputs(Bt, E, L, N, 21, dtype)
    perm = torch.from_numpy(np.random.RandomState(3).permutation(L))
    ref, ref_last = c_oracle.scan_fwd(f32["u"], f32["delta"], f32["A"], f32["B"], f32["C"], f32["D"],
                                      np.ascontiguousarray(f32["z"][:, :, perm.numpy()]), f32["delta_bias"], True)
    out, last, ckpt, _ = _scan_fwd(d["u"], d["delta"], d["A"], d["B"], d["C"], d["D"], d["z"], d["delta_bias"], True,
                                   z_rowmap=perm.to(DEV).to(torch.int32), want_last_state=True, want_ckpt=True)
    check_close(out, ref, f"scan tma {dtype} {shape}", rtol=rtol, atol=1e-5, max_strict_viol=1.0)
    check_close(last, ref_last, f"scan tma {dtype} {shape} last_state", max_strict_viol=1e-3)
    check_close(ckpt[:, -1], ref_last, f"scan tma {dtype} {shape} last checkpoint", max_strict_viol=1e-3)
    # no z, no D, no bias, no softplus
    ref2, _ = c_oracle.scan_fwd(f32["u"], f32["delta"], f32["A"], f32["B"], f32["C"], None, None, None, False)
    out2, _, _, _ = _scan_fwd(d["u"], d["delta"], d["A"], d["B"], d["C"], None, None, None, False, want_last_state=False)
    check_close(out2, ref2, f"scan tma {dtype} {shape} plain", rtol=rtol, atol=1e-5, max_strict_viol=1.0)


@pytest.mark.parametrize("mode", ["3", "5", "5:4:2", "5:4:6", "5:8:0"])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_selective_scan_warp_private_pipeline_bit_identical(mode, dtype, monkeypatch):
    """ZG_SCAN_WP=3 (scan_fwd_wp2.cuh: every warp runs its own staging ring, no block barrier, two channels per lane) and 5
    (scan_fwd_wph.cuh: CTAs that mix those warps with warps of one channel per lane) against ZG_SCAN_WP=0 (scan_fwd_tma_kernel):
    the same operations in the same order per channel, so every output -- out, last state, checkpoints (which both settings
    leave to the CTA-wide kernel), the reversed / accumulated output of the v2 sweep, the two-level z batch -- is bit identical.
    (The CTA-wide kernel itself is checked against the C oracle by the tests above and below.)"""
    from zigma_b200.selective_scan_interface import _scan_fwd
    N = 16
    if ":" in mode:     # mixed CTAs with another split than the default 8 wide + 2 narrow warps (scan_auto_choice picks these too)
        mode, nd, ns = mode.split(":")
        monkeypatch.setenv("ZG_SCAN_WPH_ND", nd)
        monkeypatch.setenv("ZG_SCAN_WPH_NS", ns)

    def both(fn):
        monkeypatch.setenv("ZG_SCAN_WP", "0")
        a = fn()
        monkeypatch.setenv("ZG_SCAN_WP", mode)
        b = fn()
        torch.cuda.synchronize()
        return a, b

    def same(a, b, what):
        for i, (x, y) in enumerate(zip(a, b)):
            if x is None or not torch.is_tensor(x):
                continue
            assert torch.equal(x, y), f"{what}: output {i} differs, max|diff| {(x.float() - y.float()).abs().max().item():.3e}"

    for shape, G in (((2, 192, 264), 1), ((3, 64, 8), 1), ((1, 128, 1024), 1), ((2, 256, 40), 2), ((5, 320, 16), 1)):
        Bt, E, L = shape
        inp = synth.synth_scan_inputs(Bt, E, L, N, G, seed=41 + L)
        d = {k: (v.to(dtype) if k in ("u", "delta", "z", "B", "C") else v).to(DEV) for k, v in inp.items()}
        tm = lambda x: x.transpose(1, 2).contiguous().transpose(1, 2)
        u, dl, z = tm(d["u"]), tm(d["delta"]), tm(d["z"])
        Bv, Cv = d["B"].transpose(2, 3).contiguous().transpose(2, 3), d["C"].transpose(2, 3).contiguous().transpose(2, 3)
        perm = torch.from_numpy(np.random.RandomState(3).permutation(L)).to(DEV).to(torch.int32)
        # the model's call: z gathered through the table, D, bias, softplus, last state, checkpoints
        same(*both(lambda: _scan_fwd(u, dl, d["A"], Bv, Cv, d["D"], z, d["delta_bias"], True, z_rowmap=perm, want_last_state=True, want_ckpt=True)),
             f"wp {mode} {dtype} {shape} full")
        same(*both(lambda: _scan_fwd(u, dl, d["A"], Bv, Cv, d["D"], z, d["delta_bias"], True, want_last_state=False)), f"wp {mode} {dtype} {shape} z in order")
        same(*both(lambda: _scan_fwd(u, dl, d["A"], Bv, Cv, None, None, None, False, want_last_state=True)), f"wp {mode} {dtype} {shape} bare")
        # second sweep of scan_type v2: reversed and accumulated into an existing output
        P = torch.randn(Bt, L, E, device=DEV).to(dtype)

        def sweep2():
            buf = P.clone()
            _scan_fwd(u, dl, d["A"], Bv, Cv, d["D"], z, d["delta_bias"], True, want_last_state=False, out=buf.transpose(1, 2), out_reverse=True, out_accumulate=True)
            return (buf,)
        same(*both(sweep2), f"wp {mode} {dtype} {shape} reverse + accumulate")
    # two-level z batch of the temporal video layers
    Bt, T, K, E = 2, 16, 8, 128
    xz = torch.randn(Bt, T * K, 2 * E, device=DEV).to(dtype)
    inp = synth.synth_scan_inputs(Bt * K, E, T, N, 1, seed=33)
    d = {k: (v.to(dtype) if k in ("u", "delta", "B", "C") else v).to(DEV) for k, v in inp.items()}
    tm = lambda x: x.transpose(1, 2).contiguous().transpose(1, 2)
    Bv, Cv = d["B"].transpose(2, 3).contiguous().transpose(2, 3), d["C"].transpose(2, 3).contiguous().transpose(2, 3)
    z_btk = xz.view(Bt, T, K, 2 * E)[:, :, :, E:]
    perm = torch.randperm(T, device=DEV).to(torch.int32)
    same(*both(lambda: _scan_fwd(tm(d["u"]), tm(d["delta"]), d["A"], Bv, Cv, d["D"], None, d["delta_bias"], True, z_rowmap=perm, want_last_state=False, z_btk=z_btk)),
         f"wp {mode} {dtype} z_btk")


@pytest.mark.parametrize("wp", ["3", "5"])
def test_selective_scan_warp_private_pipeline_vs_oracle(wp):
    """The hot-path scan tests (C oracle, zigzag table, v2 sweep, temporal layout) with ZG_SCAN_WP set, in a child process."""
    import os, subprocess, sys
    from util import ROOT
    env = dict(os.environ, ZG_SCAN_WP=wp)
    r = subprocess.run([sys.executable, "-m", "pytest", os.path.join(ROOT, "tests", "test_gpu_ops.py"), "-m", "gpu", "-q", "-x", "-p", "no:cacheprovider",
                        "-k", "tma_pipeline or out_reverse or temporal_layout or z_rowmap"], capture_output=True, text=True, cwd=ROOT, env=env, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-1000:]


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_selective_scan_out_reverse_accumulate(dtype):
    """ZG_SCAN_OUT_REVERSE | ZG_SCAN_OUT_ACCUMULATE: the kernel writes step l to position L-1-l and adds into `out` with the
    rounding of an eager 16-bit `a + b` -- exactly `P + y.flip(-1)` of mamba_simple.py:337, bit for bit."""
    from zigma_b200.selective_scan_interface import _scan_fwd
    Bt, E, L, N = 2, 128, 72, 16
    d, _ = _tok_inputs(Bt, E, L, N, 31, dtype)
    y, _, _, _ = _scan_fwd(d["u"], d["delta"], d["A"], d["B"], d["C"], d["D"], d["z"], d["delta_bias"], True, want_last_state=False)
    P = torch.randn(Bt, L, E, device=DEV).to(dtype)
    buf = P.clone()
    out, _, _, _ = _scan_fwd(d["u"], d["delta"], d["A"], d["B"], d["C"], d["D"], d["z"], d["delta_bias"], True, want_last_state=False,
                             out=buf.transpose(1, 2), out_reverse=True, out_accumulate=True)
    assert out.data_ptr() == buf.data_ptr()
    want = P + y.transpose(1, 2).flip(1)                     # eager 16-bit add of the flipped result
    assert torch.equal(buf, want)
    rev = torch.empty_like(buf)
    _scan_fwd(d["u"], d["delta"], d["A"], d["B"], d["C"], d["D"], d["z"], d["delta_bias"], True, want_last_state=False,
              out=rev.transpose(1, 2), out_reverse=True)
    assert torch.equal(rev, y.transpose(1, 2).flip(1))
    with pytest.raises(RuntimeError):                        # fp32 / other shapes: an error, never a silently ignored flag
        f = {k: (v.float() if v.dtype == dtype else v) for k, v in d.items()}
        _scan_fwd(f["u"], f["delta"], f["A"], f["B"], f["C"], f["D"], f["z"], f["delta_bias"], True, want_last_state=False,
                  out=torch.zeros(Bt, L, E, device=DEV).transpose(1, 2), out_reverse=True, out_accumulate=True)


@pytest.mark.parametrize("dtype,rtol", [(torch.bfloat16, 1.6e-2), (torch.float16, 2e-3)])
@pytest.mark.parametrize("R,E", [(40, 128), (48, 192)])
def test_selective_scan_fused_dt_proj(dtype, rtol, R, E):
    """Fused dt_proj prologue (zg_scan_params.dt_w): delta = round(dt_w @ x_dbl[:, :R]) formed inside the scan kernel on the
    tensor cores, B / C read from the same x_dbl rows (selective_scan_interface.py:322-326 of the reference).  The dt inputs are
    dyadic rationals, so the fp32 accumulation is exact in any order and delta rounds identically in kernel and oracle."""
    from zigma_b200.selective_scan_interface import _scan_fwd
    Bt, L, N = 2, 136, 16
    d, f32 = _tok_inputs(Bt, E, L, N, 23, dtype)
    rs = np.random.RandomState(5)
    xdt = torch.from_numpy(rs.randint(-16, 17, size=(Bt, L, R)).astype(np.float32) / 8)
    wdt = torch.from_numpy(rs.randint(-8, 9, size=(E, R)).astype(np.float32) / 64)
    delta = torch.einsum("blr,er->bel", xdt, wdt).to(dtype)                 # exact sums, one rounding
    x_dbl = torch.cat([xdt, torch.from_numpy(f32["B"][:, 0]).permute(0, 2, 1), torch.from_numpy(f32["C"][:, 0]).permute(0, 2, 1)], dim=2).to(dtype).to(DEV)
    Bv = x_dbl[:, :, R:R + N].permute(0, 2, 1).unsqueeze(1)
    Cv = x_dbl[:, :, R + N:].permute(0, 2, 1).unsqueeze(1)
    perm = torch.from_numpy(np.random.RandomState(4).permutation(L))
    ref, ref_last = c_oracle.scan_fwd(f32["u"], delta.float().numpy(), f32["A"], f32["B"], f32["C"], f32["D"],
                                      np.ascontiguousarray(f32["z"][:, :, perm.numpy()]), f32["delta_bias"], True)
    out, last, _, _ = _scan_fwd(d["u"], None, d["A"], Bv, Cv, d["D"], d["z"], d["delta_bias"], True, z_rowmap=perm.to(DEV).to(torch.int32),
                                want_last_state=True, dt_proj=(wdt.to(dtype).to(DEV), x_dbl))
    check_close(out, ref, f"scan fused dt_proj {dtype} R={R}", rtol=rtol, atol=1e-5, max_strict_viol=1.0)
    check_close(last, ref_last, f"scan fused dt_proj {dtype} R={R} last_state", max_strict_viol=1e-3)
    # same result as the two-kernel route (GEMM, then scan on the materialised delta), bit for bit
    d_log = delta.to(DEV).transpose(1, 2).contiguous().transpose(1, 2)
    out_u, _, _, _ = _scan_fwd(d["u"], d_log, d["A"], Bv, Cv, d["D"], d["z"], d["delta_bias"], True, z_rowmap=perm.to(DEV).to(torch.int32), want_last_state=False)
    assert torch.equal(out, out_u)
    # a request that does not fit the prologue is an error, not a silent fallback
    with pytest.raises(RuntimeError):
        _scan_fwd(d["u"][:, :, :12], None, d["A"], Bv[..., :12], Cv[..., :12], d["D"], d["z"][:, :, :12], d["delta_bias"], True,
                  dt_proj=(wdt.to(dtype).to(DEV), x_dbl[:, :12]))


def test_selective_scan_properties_full_size():
    """BASELINE config-2 layer shape (bs=64, E=1280, L=1024, N=16, bf16, token-major): too big for
    the CPU oracle in seconds, so size-independent properties instead:
      * causality: the first half of the output does not depend on the second half of the inputs;
      * batch independence + determinism: a batch slice recomputed alone is bit-identical;
      * a random subset of (b, e) rows equals the C oracle run on just those rows."""
    from zigma_b200 import selective_scan_fn
    Bt, E, L, N = 64, 1280, 1024, 16
    gen = torch.Generator(device=DEV).manual_seed(0)
    rnd = lambda *s: torch.randn(*s, device=DEV, generator=gen)
    u, z = rnd(Bt, L, E).bfloat16(), rnd(Bt, L, E).bfloat16()
    delta = (0.5 * torch.rand(Bt, L, E, device=DEV, generator=gen)).bfloat16()
    xbc = rnd(Bt, L, 2 * N).bfloat16()
    A = -0.5 * torch.rand(E, N, device=DEV, generator=gen)
    D, bias = rnd(E), 0.5 * torch.rand(E, device=DEV, generator=gen)
    lg = lambda x: x.transpose(1, 2)
    Bv = xbc[:, :, :N].permute(0, 2, 1).unsqueeze(1)
    Cv = xbc[:, :, N:].permute(0, 2, 1).unsqueeze(1)
    run = lambda u_, d_, z_, B_, C_: selective_scan_fn(lg(u_), lg(d_), A, B_, C_, D, z=lg(z_), delta_bias=bias, delta_softplus=True)
    import os
    from zigma_b200 import _lib
    out = run(u, delta, z, Bv, Cv)
    assert out.shape == (Bt, E, L) and torch.isfinite(out.float()).all()
    auto = "ZG_SCAN_WP" not in os.environ
    if auto:    # scan_auto_choice: 5120 units on this device's SMs (132 SMs -> 32-channel warps)
        mode = _lib.scan_kernel_choice(Bt, E, sms=torch.cuda.get_device_properties(0).multi_processor_count)[0]
        want = {0: "scan_fwd_tma_kernel", 3: "scan_fwd_wp2_kernel", 5: "scan_fwd_wph_kernel"}[mode]
        assert mode in (3, 5) and want in _lib.last_scan_kernel(), _lib.last_scan_kernel()
    # causality
    u2, d2, z2, x2 = u.clone(), delta.clone(), z.clone(), xbc.clone()
    u2[:, L // 2:] = 0; d2[:, L // 2:] = 0; z2[:, L // 2:] = 1; x2[:, L // 2:] = 0
    out2 = run(u2, d2, z2, x2[:, :, :N].permute(0, 2, 1).unsqueeze(1), x2[:, :, N:].permute(0, 2, 1).unsqueeze(1))
    assert torch.equal(out[:, :, : L // 2], out2[:, :, : L // 2])
    # batch slice, bit identical
    sl = slice(17, 19)
    out3 = run(u[sl].contiguous(), delta[sl].contiguous(), z[sl].contiguous(),
               xbc[sl].contiguous()[:, :, :N].permute(0, 2, 1).unsqueeze(1), xbc[sl].contiguous()[:, :, N:].permute(0, 2, 1).unsqueeze(1))
    assert torch.equal(out[sl], out3)
    if auto:    # ... and two batch rows are the CTA-wide kernel's: the comparison above is ACROSS the two kernels
        assert "scan_fwd_tma_kernel" in _lib.last_scan_kernel(), _lib.last_scan_kernel()
    # sampled rows vs the C oracle
    bs, es = [0, 31, 63], [0, 5, 640, 1279]
    f = lambda x: x[bs][:, :, es].float().cpu().permute(0, 2, 1).contiguous().numpy()
    ref, _ = c_oracle.scan_fwd(f(u), f(delta), A[es].cpu().numpy(), xbc[bs][:, :, :N].float().cpu().permute(0, 2, 1).unsqueeze(1).contiguous().numpy(),
                               xbc[bs][:, :, N:].float().cpu().permute(0, 2, 1).unsqueeze(1).contiguous().numpy(),
                               D[es].cpu().numpy(), f(z), bias[es].cpu().numpy(), True)
    check_close(out[bs][:, es].float(), ref, "full-size sampled rows vs C oracle (bf16 out)", rtol=1.6e-2, atol=1e-5, max_strict_viol=1.0)


def test_selective_scan_rejects_bad_input():
    from zigma_b200 import selective_scan_fn
    u = torch.randn(1, 4, 8, device=DEV)
    A = -torch.rand(4, 2, device=DEV)
    Bm = torch.randn(1, 2, 8, device=DEV)
    with pytest.raises(RuntimeError):
        selective_scan_fn(u, u[:, :, :4], A, Bm, Bm)                       # delta shape
    with pytest.raises(RuntimeError):
        selective_scan_fn(u, u, A.half(), Bm, Bm)                          # A dtype
    with pytest.raises(RuntimeError):
        selective_scan_fn(u, u, -torch.rand(4, 65, device=DEV), torch.randn(1, 65, 8, device=DEV), torch.randn(1, 65, 8, device=DEV))


# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("channel_last", [False, True])
def test_causal_conv1d_golden_fp32(channel_last):
    from zigma_b200 import causal_conv1d_fn
    g = gold("conv")
    x = t(g["x"], DEV)
    if channel_last:
        x = x.transpose(1, 2).contiguous().transpose(1, 2)
    for W in (2, 3, 4):
        for silu in (0, 1):
            for hb in (0, 1):
                tag = f"W{W}_s{silu}_b{hb}"
                out = causal_conv1d_fn(x, t(g[f"w{W}"], DEV), t(g[f"b{W}"], DEV) if hb else None, "silu" if silu else None)
                check_close(out, g["out_" + tag], f"conv {tag} cl={channel_last}")


@pytest.mark.parametrize("itype", [torch.float32, torch.float16, torch.bfloat16])
@pytest.mark.parametrize("seqlen", [8, 151, 1024, 1134])
@pytest.mark.parametrize("channel_last", [False, True])
def test_causal_conv1d_reference_test_shapes(seqlen, itype, channel_last):
    """Shapes and tolerances of dis_causal_conv1d/tests/test_causal_conv1d.py:14-75 (dim not divisible
    by 64, x sliced out of a wider tensor -> non-trivial batch stride)."""
    from zigma_b200 import causal_conv1d_fn
    rtol, atol = (3e-4, 1e-3) if itype == torch.float32 else (3e-3, 5e-3)
    if itype == torch.bfloat16:
        rtol, atol = 1e-2, 5e-2
    torch.manual_seed(0)
    dim, W = 512 + 32, 4
    if not channel_last:
        x = torch.randn(2, 64 + dim + 64, seqlen, device=DEV, dtype=itype)[:, 64:64 + dim, :]
    else:
        x = torch.randn(2, seqlen, 64 + dim + 64, device=DEV, dtype=itype)[:, :, 64:64 + dim].transpose(1, 2)
    w = torch.randn(dim, W, device=DEV, dtype=torch.float32)
    b = torch.randn(dim, device=DEV, dtype=torch.float32)
    out = causal_conv1d_fn(x, w, b, activation="silu")
    ref = zo.causal_conv1d(x.cpu(), w.cpu(), b.cpu(), "silu")
    assert out.dtype == itype and out.shape == x.shape
    assert torch.allclose(out.cpu().float(), ref.float(), rtol=rtol, atol=atol), (out.cpu().float() - ref.float()).abs().max()


def test_causal_conv1d_rowmap_fuses_permutation():
    from zigma_b200.causal_conv1d_interface import _conv_fwd
    import zigma_b200
    Bt, E, L = 2, 128, 64
    perm = torch.from_numpy(zigma_b200.zigzag_path(8)[5])
    xz = torch.randn(Bt, L, 2 * E, device=DEV).bfloat16()
    w, b = torch.randn(E, 4, device=DEV).bfloat16(), torch.randn(E, device=DEV).bfloat16()
    x_log = xz[:, :, :E].transpose(1, 2)
    out = _conv_fwd(x_log, w, b, True, x_rowmap=perm.to(DEV).to(torch.int32))
    # fp32 math on the bf16 inputs, one rounding at the end (what causal_conv1d_fwd.cu:103-118 does)
    ref = zo.causal_conv1d(xz[:, :, :E].transpose(1, 2)[:, :, perm.to(DEV)].cpu(), w.cpu().float(), b.cpu().float(), "silu")
    check_close(out, ref, "conv x_rowmap (bf16)", rtol=8e-3, atol=1e-5, max_strict_viol=1.0)


def test_conv_segments_and_scan_two_level_z_batch_temporal_layout():
    """The two kernel features behind the copy-free temporal video layers (engine._core_temporal; mamba_simple.py:416-442):
    (a) causal_conv1d with x_rowmap + seg_len: a (b, t k) token-major tensor convolved as (b k) sequences of T positions, taps
        never crossing a segment start -- against the oracle conv on the explicitly permuted (b k, E, T) tensor;
    (b) selective_scan with z_btk: sequence b K + k gates with z[b, perm[t], k, :] -- against the oracle scan on the explicitly
        gathered z."""
    from zigma_b200.causal_conv1d_interface import _conv_fwd
    from zigma_b200.selective_scan_interface import _scan_fwd
    dtype = torch.bfloat16
    Bt, T, K, E, N = 2, 16, 8, 128, 16
    L = T * K
    gen = torch.Generator(device=DEV).manual_seed(9)
    xz = torch.randn(Bt, L, 2 * E, device=DEV, generator=gen).to(dtype)               # (b, t k) token-major, x | z halves
    w = (0.5 * torch.randn(E, 4, device=DEV, generator=gen)).to(dtype)
    bias = (0.1 * torch.randn(E, device=DEV, generator=gen)).to(dtype)
    perm = torch.randperm(T, device=DEV, generator=gen)
    k_idx = torch.arange(K, device=DEV)
    comp_in = (perm.view(1, T) * K + k_idx.view(K, 1)).reshape(-1).to(torch.int32)    # [k T + t] -> perm[t] K + k
    xc = _conv_fwd(xz[:, :, :E].transpose(1, 2), w, bias, True, x_rowmap=comp_in, seg_len=T)     # (Bt, E, L) logical, (k, t) order
    x_perm = xz[:, :, :E].view(Bt, T, K, E)[:, perm].permute(0, 2, 3, 1).reshape(Bt * K, E, T)   # explicit (b k, E, t) gather
    want = zo.causal_conv1d(x_perm.float().cpu(), w.float().cpu(), bias.float().cpu(), "silu")
    got = xc.transpose(1, 2).reshape(Bt, K, T, E).permute(0, 1, 3, 2).reshape(Bt * K, E, T)
    check_close(got, want, "conv seg_len + composite rowmap", rtol=1.6e-2, atol=1e-5, max_strict_viol=1.0)
    # (b) scan over the (b k) sequences, z through the two-level batch
    inp = synth.synth_scan_inputs(Bt * K, E, T, N, 1, seed=33)
    lo = {kk: (v.to(dtype) if kk in ("u", "delta", "B", "C") else v) for kk, v in inp.items()}
    d = {kk: v.to(DEV) for kk, v in lo.items()}
    tm = lambda x: x.transpose(1, 2).contiguous().transpose(1, 2)
    Bv, Cv = d["B"].transpose(2, 3).contiguous().transpose(2, 3), d["C"].transpose(2, 3).contiguous().transpose(2, 3)
    z_btk = xz.view(Bt, T, K, 2 * E)[:, :, :, E:]
    out, _, _, _ = _scan_fwd(tm(d["u"]), tm(d["delta"]), d["A"], Bv, Cv, d["D"], None, d["delta_bias"], True,
                             z_rowmap=perm.to(torch.int32), want_last_state=False, z_btk=z_btk)
    z_perm = z_btk[:, perm].permute(0, 2, 3, 1).reshape(Bt * K, E, T)                  # z[b, perm[t], k, :] as (b k, E, t)
    f = lambda v: v.float().cpu().numpy()
    ref, _ = c_oracle.scan_fwd(f(lo["u"]), f(lo["delta"]), f(lo["A"]), f(lo["B"]), f(lo["C"]), f(lo["D"]), f(z_perm), f(lo["delta_bias"]), True)
    check_close(out, ref, "scan z_btk (two-level z batch)", rtol=1.6e-2, atol=1e-5, max_strict_viol=1.0)
    with pytest.raises(RuntimeError):        # seg_len outside the fast path is an error, not silently ignored
        _conv_fwd(xz[:, :, :E].transpose(1, 2).float(), w.float(), bias.float(), True, x_rowmap=comp_in, seg_len=T)


def test_causal_conv1d_backward_golden():
    from zigma_b200 import causal_conv1d_fn
    g = gold("conv")
    for tag in ("W4_s1_b1", "W3_s0_b0", "W2_s1_b0"):
        W, silu, hb = int(tag[1]), int(tag[4]), int(tag[7])
        x = t(g["x"], DEV).requires_grad_()
        w = t(g[f"w{W}"], DEV).requires_grad_()
        b = t(g[f"b{W}"], DEV).requires_grad_() if hb else None
        out = causal_conv1d_fn(x, w, b, "silu" if silu else None)
        out.backward(t(g["g"], DEV))
        check_close(x.grad, g["dx_" + tag], "conv dx " + tag)
        check_close(w.grad, g["dw_" + tag], "conv dweight " + tag, rtol=1e-3, atol=1e-4)
        if hb:
            check_close(b.grad, g["db_" + tag], "conv dbias " + tag, rtol=1e-3, atol=1e-4)


def test_causal_conv1d_backward_token_major_and_rowmap():
    """Token-major backward kernel: (a) same golden gradients as the channel-first kernel when the tensors are
    handed over channel-last; (b) with x_rowmap it equals gather -> conv backward -> scatter, odd sizes
    (dim not a multiple of 4, seqlen not a multiple of the 64-position chunk) included."""
    from zigma_b200 import causal_conv1d_fn
    from zigma_b200.causal_conv1d_interface import _conv_bwd
    g = gold("conv")
    tm = lambda a: a.transpose(1, 2).contiguous().transpose(1, 2)
    for tag in ("W4_s1_b1", "W3_s0_b0", "W2_s1_b0"):
        W, silu, hb = int(tag[1]), int(tag[4]), int(tag[7])
        x = tm(t(g["x"], DEV)).requires_grad_()
        w = t(g[f"w{W}"], DEV).requires_grad_()
        b = t(g[f"b{W}"], DEV).requires_grad_() if hb else None
        out = causal_conv1d_fn(x, w, b, "silu" if silu else None)
        out.backward(tm(t(g["g"], DEV)))
        check_close(x.grad, g["dx_" + tag], "conv dx (token-major) " + tag)
        check_close(w.grad, g["dw_" + tag], "conv dweight (token-major) " + tag, rtol=1e-3, atol=1e-4)
        if hb:
            check_close(b.grad, g["db_" + tag], "conv dbias (token-major) " + tag, rtol=1e-3, atol=1e-4)
    gen = torch.Generator(device=DEV).manual_seed(4)
    # (the last three shapes take the branch-free 16-bit fast path: whole 32-position chunks; one without a rowmap, one with
    # a single chunk per row, i.e. no halo at all)
    for (bs, E, L, dt, use_map) in ((2, 64, 200, torch.float32, True), (3, 30, 77, torch.float32, True), (2, 128, 256, torch.bfloat16, True),
                                    (3, 96, 96, torch.float16, False), (5, 64, 32, torch.bfloat16, True)):
        x = tm(torch.randn(bs, E, L, device=DEV, generator=gen).to(dt))
        do = tm(torch.randn(bs, E, L, device=DEV, generator=gen).to(dt))
        w = torch.randn(E, 4, device=DEV, generator=gen).to(dt)
        b = torch.randn(E, device=DEV, generator=gen).to(dt)
        perm = torch.randperm(L, device=DEV, generator=gen) if use_map else torch.arange(L, device=DEV)
        dx, dw, db = _conv_bwd(x, w, b, do, True, x_rowmap=perm.to(torch.int32) if use_map else None)
        # reference: autograd through the ORACLE's causal_conv1d (zo.causal_conv1d, causal_conv1d_interface.py:49-65 of the
        # reference) applied to the gathered sequence -- the gather's own backward scatters dx back
        xr = x.float().cpu().contiguous().requires_grad_()
        wr, br = w.float().cpu().requires_grad_(), b.float().cpu().requires_grad_()
        zo.causal_conv1d(xr[:, :, perm.cpu()], wr, br, "silu").backward(do.float().cpu().contiguous())
        want_dx, dwr, dbr = xr.grad, wr.grad, br.grad
        lo = dt != torch.float32
        check_close(dx, want_dx, f"conv dx rowmap {bs}x{E}x{L}", **(dict(rtol=2e-2, atol=2e-2, max_strict_viol=1.0) if lo else {}))
        check_close(dw, dwr, f"conv dweight rowmap {bs}x{E}x{L}", rtol=1e-3, atol=1e-4, max_strict_viol=1.0 if lo else 1e-4)
        check_close(db, dbr, f"conv dbias rowmap {bs}x{E}x{L}", rtol=1e-3, atol=1e-4, max_strict_viol=1.0 if lo else 1e-4)


# ------------------------------------------------------------------------------------------------
def test_add_norm_golden():
    from zigma_b200 import rms_norm_fn, layer_norm_fn
    g = gold("norm")
    x, res, w, b = (t(g[k], DEV) for k in ("x", "res", "w", "b"))
    for rms in (1, 0):
        for hr in (1, 0):
            fn = rms_norm_fn if rms else layer_norm_fn
            y, r = fn(x, w, None if rms else b, residual=res if hr else None, prenorm=True, residual_in_fp32=True, eps=1e-5)
            check_close(y, g[f"y_rms{rms}_res{hr}"], f"norm rms={rms} res={hr} y")
            check_close(r, g[f"r_rms{rms}_res{hr}"], f"norm rms={rms} res={hr} residual")
    y, r = rms_norm_fn(x.bfloat16(), w.bfloat16(), None, residual=res, prenorm=True, residual_in_fp32=True, eps=1e-5)
    assert y.dtype == torch.bfloat16 and r.dtype == torch.float32
    check_close(y, g["y_bf16"], "norm bf16 y", rtol=8e-3, max_strict_viol=1.0)
    check_close(r, g["r_bf16"], "norm bf16 residual")


@pytest.mark.parametrize("lch", ["16", "32", "64"])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_causal_conv1d_smem_staged_kernel_bit_identical(lch, dtype, monkeypatch):
    """ZG_CONV_SMEM=1 (conv_fwd_tok8s_kernel: 8 channels per lane, rows staged through a per-lane cp.async ring) against the default
    token-major kernel (conv_fwd_tok4_kernel, itself checked against the oracle above): same taps in the same order -> same bits.
    Plain rows, rows gathered through a table, and independent segments (the temporal video layers)."""
    from zigma_b200.causal_conv1d_interface import _conv_fwd
    torch.manual_seed(5)
    for Bt, L, E, seg in ((3, 128, 256, 0), (2, 192, 768, 0), (2, 256, 512, 16), (1, 64, 1280, 0)):
        xz = torch.randn(Bt, L, 2 * E, device=DEV).to(dtype)
        w, b = torch.randn(E, 4, device=DEV).to(dtype), torch.randn(E, device=DEV).to(dtype)
        perm = torch.from_numpy(np.random.RandomState(7).permutation(L)).to(DEV).to(torch.int32)
        for rowmap in (None, perm):
            outs = []
            for flag in ("0", "1"):
                monkeypatch.setenv("ZG_CONV_SMEM", flag)
                monkeypatch.setenv("ZG_CONV_SMEM_LCH", lch)
                outs.append(_conv_fwd(xz[:, :, :E].transpose(1, 2), w, b, True, x_rowmap=rowmap, seg_len=seg).clone())
            torch.cuda.synchronize()
            assert torch.equal(outs[0], outs[1]), f"{dtype} lch {lch} {(Bt, L, E, seg)} rowmap {rowmap is not None}: max|diff| {(outs[0].float() - outs[1].float()).abs().max().item():.3e}"
    # and against the oracle directly (fp32 math on the rounded inputs)
    monkeypatch.setenv("ZG_CONV_SMEM", "1")
    x = torch.randn(2, 512, 128, device=DEV).to(dtype)       # (B, E, L) logical, token-major memory
    xt = x.transpose(1, 2).contiguous().transpose(1, 2)
    w, b = torch.randn(512, 4, device=DEV).to(dtype), torch.randn(512, device=DEV).to(dtype)
    got = _conv_fwd(xt, w, b, True)
    ref = zo.causal_conv1d(x.float().cpu(), w.float().cpu(), b.float().cpu(), "silu")
    check_close(got, ref, f"conv smem-staged kernel vs oracle {dtype}", rtol=8e-3, max_strict_viol=1.0)


def test_block_tail_pos_embed_fold_matches_separate_add():
    """zg_block_tail_fwd_pe (first tail, positional embedding as a broadcast mix table, no gate) is bit-identical to the eager
    `tokens + pos_embed` (model_zigma.py:941) followed by the plain first tail, and agrees with the oracle's add + RMSNorm."""
    from zigma_b200.engine import block_tail
    for dtype, D in ((torch.bfloat16, 640), (torch.float16, 768), (torch.float32, 64), (torch.bfloat16, 1536)):
        torch.manual_seed(11)
        Bt, L = 3, 48
        tok, pe = torch.randn(Bt, L, D).to(dtype), (0.5 * torch.randn(1, L, D)).to(dtype)
        mods = (0.3 * torch.randn(Bt, 3 * D)).to(dtype)
        nw = (1 + 0.1 * torch.randn(D)).to(dtype)
        md, nwd = mods.to(DEV), nw.to(DEV)
        r0, n0, m0 = block_tail((tok.to(DEV) + pe.to(DEV)).contiguous(), None, None, md[:, :D], md[:, D:2 * D], nwd, None, None, 1e-5)
        r1, n1, m1 = block_tail(tok.to(DEV), pe.to(DEV).reshape(L, D), None, md[:, :D], md[:, D:2 * D], nwd, None, None, 1e-5, mix_bcast=True)
        assert torch.equal(r0, r1) and torch.equal(n0, n1) and torch.equal(m0, m1), f"{dtype} D={D}"
        normed_ref, res_ref = zo.add_norm(tok + pe, nw, None, None, True, True, 1e-5, True)
        check_close(r1, res_ref, f"block_tail_pe residual {dtype}")
        check_close(n1, normed_ref, f"block_tail_pe normed {dtype}", **(dict(rtol=1e-3) if dtype == torch.float32 else dict(rtol=8e-3, max_strict_viol=1.0)))
    with pytest.raises(RuntimeError):      # the table takes no gate
        block_tail(tok.to(DEV), pe.to(DEV).reshape(L, D), md[:, :D], md[:, :D], md[:, :D], nwd, None, None, 1e-5, mix_bcast=True)
