"""GPU (H100): stochastic depth inside the fused block tail (zg_block_tail_fwd_dp / zg_block_tail_bwd_dp and the _det twin).

* every drop-path instantiation against an fp64 restatement, with the bounds and helpers of test_gpu_norm_kernels.py;
* path_scale == 1 gives the plain entry points' bits, a dropped sample gives exact zeros;
* the kernels a train-mode model launches (profiler), and train mode vs the per-op block loop on the same seed;
* train-mode training steps repeat bit for bit under torch.use_deterministic_algorithms (tests/_droppath_det_worker.py)."""
import os
import re
import subprocess
import sys

import pytest
import torch

from test_gpu_norm_kernels import (DTYPES, LOWP, _NAME, _deterministic, _rd, _tail_inputs, check_colsum, check_elem, ref_gated,
                                   ref_modulate, ref_tail_bwd)
from util import ROOT, check_close

pytestmark = pytest.mark.gpu
DEV = "cuda"
WIDTHS = (36, 368, 640, 768, 1024)               # forward Q 1, 1, 2, 2, 2; backward MAXQ 4, 4, 5, 6, 8
B, L, EPS = 6, 37, 1e-5


def masks(T):
    """(name, s) pairs: 0 or round_T(1 / keep) per sample for keep 0.5 / 0.9 / 0.998, every sample dropped, none dropped."""
    out = []
    for keep in (0.5, 0.9, 0.998):
        v = torch.tensor(1.0, dtype=T).div_(keep)          # as DropPath.draw forms it
        out.append((f"keep{keep}", (torch.tensor([0, 1, 1, 0, 1, 0], dtype=T) * v).to(T)))
    out.append(("all_dropped", torch.zeros(B, dtype=T)))
    out.append(("none_dropped", torch.full((B,), torch.tensor(1.0, dtype=T).div_(0.9).item(), dtype=T)))
    return out


def _run(T, D, s, rowmap_on, det, seed, grads_seed=None, path=True):
    """block_tail_fn forward + backward with path_scale s (None: the plain entry points).  Returns inputs and results."""
    from zigma_b200.block_ops import block_tail_fn
    x, mix, res, mods, nw, perm = _tail_inputs(B, L, D, T, seed=seed)
    g = torch.Generator().manual_seed(seed + 1 if grads_seed is None else grads_seed)
    grads = {n: torch.randn(B, L, D, generator=g).to(torch.float32 if n == "d_residual_out" else T)
             for n in ("d_residual_out", "d_normed", "d_modded")}
    md = mods.to(DEV).requires_grad_()
    dshift, dscale, dgate = md.chunk(3, dim=1)
    xd, nwd, mixd, resd = (t.to(DEV).requires_grad_() for t in (x, nw, mix, res))
    rowmap = perm.to(DEV).to(torch.int32) if rowmap_on else None
    ps = s.to(DEV) if (path and s is not None) else None
    with _deterministic(det):
        r_out, normed, modded = block_tail_fn(xd, mixd, dgate, dshift, dscale, nwd, resd, rowmap, EPS, ps)
        torch.autograd.backward([r_out, normed, modded], [grads[n].to(DEV) for n in ("d_residual_out", "d_normed", "d_modded")])
    return dict(x=x, mix=mix, res=res, mods=mods, nw=nw, perm=perm, grads=grads, r_out=r_out, normed=normed, modded=modded,
                dx=xd.grad, dmix=mixd.grad, dres=resd.grad, dmods=md.grad, dnw=nwd.grad)


def _check(T, D, name, s, rowmap_on, det, o):
    tag = f"dp {_NAME[T]} D={D} {name} rowmap={rowmap_on} det={det}"
    sd = s.double()[:, None, None]
    x, mix, res, mods, nw = o["x"], o["mix"], o["res"], o["mods"], o["nw"]
    shift, scale, gate = mods[:, :D], mods[:, D:2 * D], mods[:, 2 * D:]
    src = o["perm"] if rowmap_on else torch.arange(L)
    # forward: hidden = round(x + round(gate * mix)); kept = round(hidden * s); r = residual + kept; normed; modded
    gm = _rd(gate.double()[:, None] * mix[:, src].double(), T)
    h = _rd(x.double() + gm, T)
    kept = _rd(h * sd, T)
    r = res.double() + kept
    M_r = (x.double().abs() + gm.abs()) * sd.abs() + res.double().abs()
    rstd = (r.pow(2).mean(-1, keepdim=True) + EPS).rsqrt()
    check_elem(f"{tag} residual_out", o["r_out"], r, M_r)
    check_elem(f"{tag} normed", o["normed"], r * rstd * nw.double(), M_r * rstd * nw.double().abs(), max_ulp=2)
    check_elem(f"{tag} modded", o["modded"], *ref_modulate(o["normed"], shift, scale, T), max_ulp=2)
    # backward
    gr = o["grads"]
    ref = ref_tail_bwd(o["r_out"].detach().cpu(), nw, (shift, scale, gate), gr["d_residual_out"], gr["d_normed"], gr["d_modded"], EPS, T)
    check_elem(f"{tag} d_residual_in", o["dres"], ref["dr"], ref["M_dr"])
    check_elem(f"{tag} dx", o["dx"], ref["dh"] * sd, ref["M_dr"] * sd.abs(), max_ulp=2)      # dh = round(dr), then * s
    e_mix, M_mix, e_gate, S_gate = ref_gated(o["dx"], gate, mix[:, src])
    d_mix, M_d_mix = torch.empty_like(e_mix), torch.empty_like(e_mix)
    d_mix[:, src], M_d_mix[:, src] = e_mix, M_mix
    check_elem(f"{tag} d_mix", o["dmix"], d_mix, M_d_mix, max_ulp=2)
    dm = o["dmods"]
    check_colsum(f"{tag} dshift", dm[:, :D], ref["dshift"], ref["S_dshift"])
    check_colsum(f"{tag} dscale", dm[:, D:2 * D], ref["dscale"], ref["S_dscale"])
    check_colsum(f"{tag} dgate", dm[:, 2 * D:], e_gate, S_gate)
    check_colsum(f"{tag} d_norm_w", o["dnw"], ref["d_norm_w"], ref["S_norm_w"])
    # a dropped sample: nothing reaches hidden, the residual passes through untouched
    z = (s == 0).nonzero().flatten().tolist()
    for b in z:
        assert torch.equal(o["r_out"][b].cpu(), res[b]), tag
        assert not o["dx"][b].any() and not o["dmix"][b].any() and not dm[b, 2 * D:].any(), tag


CASES = [(T, D, rm) for T in DTYPES for D in WIDTHS for rm in (False, True)]


@pytest.mark.parametrize("T,D,rowmap_on", CASES, ids=[f"{_NAME[t]}-{d}-{'rowmap' if r else 'plain'}" for t, d, r in CASES])
def test_drop_path_tail_vs_fp64(T, D, rowmap_on):
    for k, (name, s) in enumerate(masks(T)):
        for det in (False, True):
            _check(T, D, name, s, rowmap_on, det, _run(T, D, s, rowmap_on, det, seed=11 * D + k))


@pytest.mark.parametrize("T", DTYPES, ids=[_NAME[t] for t in DTYPES])
def test_unit_scale_matches_plain_tail_bitwise(T):
    """path_scale == 1: the drop-path kernels give the plain kernels' bits (column sums with the deterministic flag on; the
    atomic path's column sums depend on the order the CTAs run in)."""
    for D in WIDTHS:
        for det in (True, False):
            ones = torch.ones(B, dtype=T)
            a = _run(T, D, ones, True, det, seed=3 * D)
            b = _run(T, D, None, True, det, seed=3 * D)
            for k in ("r_out", "normed", "modded", "dx", "dmix", "dres") + (("dmods", "dnw") if det else ()):
                assert torch.equal(a[k], b[k]), (T, D, det, k)


# ------------------------------------------------------------------------------------------------ what runs
def _kernels(prof, families):
    out = {}
    for evt in prof.events():
        if evt.device_type != torch.autograd.DeviceType.CUDA:
            continue
        m = re.search(r"zg::(\w+)<(.*)>\(", evt.name)
        if m and m.group(1) in families:
            args = tuple({"(bool)1": "true", "(bool)0": "false"}.get(a.strip(), a.strip()) for a in m.group(2).split(","))
            key = (m.group(1), tuple(re.sub(r"^\((?:int|unsigned int)\)", "", a) for a in args))
            out[key] = out.get(key, 0) + 1
    return out


def test_matrix_reaches_every_drop_path_instantiation():
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for T in DTYPES:
            for D in WIDTHS:
                for det in (False, True):
                    _run(T, D, masks(T)[0][1], False, det, seed=D)
        torch.cuda.synchronize()
    seen = set(_kernels(prof, {"block_tail_dp_fwd_kernel", "block_tail_dp_bwd_kernel"}))
    TT = ("float", "__half", "__nv_bfloat16")
    want = ({("block_tail_dp_fwd_kernel", (t, q)) for t in TT for q in ("1", "2")}
            | {("block_tail_dp_bwd_kernel", (t, q, d)) for t in TT for q in ("4", "5", "6", "8") for d in ("false", "true")})
    assert len(want) == 30 and seen == want, (sorted(want - seen), sorted(seen - want))


def test_train_mode_model_launches_drop_path_tails():
    """Depth 4, rate 0.5: blocks 2 and 3 hold a DropPath.  One train-mode forward + backward launches one DP forward and one
    DP backward for each of them, the plain tail for blocks 0 and 1, and no add+norm kernel but the one of norm_f."""
    from torch.profiler import ProfilerActivity, profile
    from zigma_b200 import ZigMa
    from zigma_b200.model_zigma import DropPath
    m = ZigMa(device=DEV, in_channels=4, embed_dim=64, depth=4, img_dim=8, patch_size=1, scan_type="zigzagN8", use_pe=2,
              drop_path_rate=0.5).train()
    assert [isinstance(b.drop_path, DropPath) for b in m.blocks] == [False, False, True, True]
    x, t = torch.randn(4, 4, 8, 8, device=DEV), torch.rand(4, device=DEV)
    m(x, t).square().mean().backward()          # warm-up
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        m(x, t).square().mean().backward()
        torch.cuda.synchronize()
    k = _kernels(prof, {"block_tail_dp_fwd_kernel", "block_tail_dp_bwd_kernel", "block_tail_row4_kernel", "block_tail_bwd_kernel",
                        "block_tail_kernel", "add_norm_fwd_kernel", "add_norm_bwd_kernel", "add_norm_bwd_vec_kernel"})
    count = lambda fam: sum(v for (f, _), v in k.items() if f == fam)
    assert count("block_tail_dp_fwd_kernel") == 2 and count("block_tail_dp_bwd_kernel") == 2, k
    assert count("block_tail_row4_kernel") == 2 and count("block_tail_bwd_kernel") == 2 and count("block_tail_kernel") == 0, k
    assert count("add_norm_fwd_kernel") == 1 and count("add_norm_bwd_kernel") + count("add_norm_bwd_vec_kernel") == 1, k


# ------------------------------------------------------------------------------------------------ model level
@pytest.mark.parametrize("name", ["tiny_zigzag8", "tiny_sweep2", "tiny_video_sst"])
def test_train_mode_fused_tail_matches_unfused_block_loop(name, monkeypatch):
    """ZigMa.forward_autograd in train mode with stochastic depth: fused tails (default) vs the per-op block loop
    (ZIGMA_FUSED_TRAIN_TAIL=0) on the same seed -- same draws (CUDA generator state after the forward), output and every
    parameter gradient with the tolerances of test_gpu_bwd.py's eval-mode comparison."""
    from oracle import synth
    from oracle.gen_golden import model_io
    from util import model_case
    from zigma_b200 import ZigMa
    from zigma_b200.model_zigma import DropPath
    _, cfg, _ = model_case(name)
    cfg = dict(cfg, depth=max(cfg["depth"], 4), drop_path_rate=0.6)       # (tiny_sweep2 has 2 blocks: neither would drop)
    m = ZigMa(device=DEV, **cfg).train()
    m.load_state_dict(synth.synth_state_dict({k: tuple(v.shape) for k, v in m.state_dict().items()}, seed=0))
    x, tt, y = model_io(cfg, 8)
    target = torch.randn((8,) + tuple(m(x.to(DEV), tt.to(DEV), None if y is None else y.to(DEV)).shape[1:]),
                         generator=torch.Generator().manual_seed(77)).to(DEV)
    drawn = []
    orig = DropPath.draw

    def spy(self, x_):
        mask = orig(self, x_)
        drawn.append(mask.flatten().cpu())
        return mask
    monkeypatch.setattr(DropPath, "draw", spy)
    res = {}
    for mode in ("1", "0"):
        monkeypatch.setenv("ZIGMA_FUSED_TRAIN_TAIL", mode)
        assert m._fused_tail_ok(torch.empty(1, 1, cfg["embed_dim"], device=DEV)) == (mode == "1")
        for p_ in m.parameters():
            p_.grad = None
        drawn.clear()
        torch.manual_seed(1234)
        out = m.forward_autograd(x.to(DEV), tt.to(DEV), None if y is None else y.to(DEV))
        rng = torch.cuda.get_rng_state()
        ((out - target) ** 2).mean().backward()
        res[mode] = (out.detach(), {k: v.grad.clone() for k, v in m.named_parameters() if v.grad is not None}, rng, list(drawn))
    assert torch.equal(res["1"][2], res["0"][2]), "the two paths left the CUDA generator in different states"
    assert len(res["1"][3]) == len(res["0"][3]) and all(torch.equal(a, b) for a, b in zip(res["1"][3], res["0"][3]))
    block_masks = res["1"][3][:-1]                # the last draw is the model-level drop_path before norm_f
    assert any((mk == 0).any() and (mk != 0).any() for mk in block_masks), "no block dropped one sample and kept another"
    check_close(res["1"][0], res["0"][0], f"{name} train-mode fused-tail forward", atol=2e-5)
    assert set(res["1"][1]) == set(res["0"][1])
    for k in res["0"][1]:
        check_close(res["1"][1][k], res["0"][1][k], f"{name} train-mode fused-tail d{k}", atol=2e-5, max_strict_viol=2e-2)


def test_train_mode_steps_are_bitwise_reproducible():
    """Two fresh processes, same seeds, deterministic flag on: identical digests of train-mode training steps at rate 0.1."""
    worker = os.path.join(ROOT, "tests", "_droppath_det_worker.py")
    runs = []
    for _ in range(2):
        r = subprocess.run([sys.executable, worker], capture_output=True, text=True, timeout=1800, cwd=ROOT)
        assert r.returncode == 0 and "DROPPATH_DET_WORKER_OK" in r.stdout, r.stdout[-3000:] + r.stderr[-6000:]
        runs.append([l for l in r.stdout.splitlines() if l.startswith("DIGEST ")])
    assert len(runs[0]) > 30
    assert runs[0] == runs[1], [(a, b) for a, b in zip(*runs) if a != b][:5]
