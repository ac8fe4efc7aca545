"""Every instantiation of the selective-scan kernels (scan_fwd*.cuh, scan_bwd*.cuh), forward and backward, against a plain fp64
restatement of the same operation, in fp32 / fp16 / bf16, with and without torch.use_deterministic_algorithms.

The references read exactly what the kernels read (inputs are drawn in the kernel's dtype and upcast) and round once, to the
output dtype.  Bounds (tests/util.py), instead of a blanket rtol:
* fp32 elements: |a - e| <= C[family] * 2^-24 * M, M = the error magnitude of the element (below), fitted per kernel family;
* 16-bit elements: at most 1 ulp of the fp64 value (2 for the accumulated output of the second v2 sweep), or, for an element
  formed by cancellation, the fp32 bound plus one ulp; and the fraction of elements that differ from round(e) stays below
  MISMATCH[dtype];
* sums (dA, dD, d(delta_bias), dB, dC): rel * S + one ulp, S = the sum of the magnitudes of the summed terms.
Magnitudes.  The forward carries E_l = a_l E_{l-1} + (1 + |delta'_l A|) a_l |h_{l-1}| + |delta'_l u_l B_l| along the recurrence
(the |delta' A| factor carries the error of exp and softplus into a), M_y = (sum_n |C_n| (E_n + |h_n|) + |D u|) |z sigma(z)|.
The backward does the same on the reverse recurrence of dh.  The CPU tests below prove the backward restatement against fp64
autograd and show that every bound rejects a kernel that drops one term.  The achieved fractions of the bounds go to
$ZIGMA_PARITY_LOG when it names a file.

The last part is the instantiation inventory: the table DEFAULT lists every zg::scan_fwd* / zg::scan_bwd* kernel of the library;
a CPU test holds it against the built library, and a GPU test checks that the matrix launches exactly DEFAULT."""
import itertools
import os
import re
import shutil
import subprocess

import pytest
import torch

from util import DTYPE_NAME, check_colsum, check_elem, ulp

DEV = "cuda"
gpu = pytest.mark.gpu
F64 = torch.float64
LOWP = (torch.float16, torch.bfloat16)
DTYPES = (torch.float32, torch.float16, torch.bfloat16)
CK = 8                      # checkpoint spacing of the forward (selective_scan_interface.CKPT_EVERY, the backward's chunk)

# fp32 constants of the elementwise bound, per kernel family: the worst |a - e| / (2^-24 M) measured on an H100 80GB HBM3
# (700 W), times at most 4 -- generic forward 20.3, CTA-wide hot path 16.1, tpc2 11.7, warp-private 5.8, generic backward 10.8,
# q4 backward 7.2.  They differ because the families meet different worst cases: only the generic and the CTA-wide kernels run
# the 277- to 4096-step rows, where the state carries the most rounding; the 16-bit kernels' fp32 outputs are the states alone.
C_FAMILY = {"fwd_generic": 64, "fwd_tma": 64, "fwd_tpc2": 44, "fwd_wp": 23, "bwd_generic": 43, "bwd_q4": 28}
SUM_REL = 1e-5
MISMATCH = {torch.float16: 5e-3, torch.bfloat16: 1e-3}


# ------------------------------------------------------------------------------------------------ fp64 references
def softplus20(x):
    """log1p(exp(x)) for x <= 20, x above (the reference's threshold)."""
    return torch.where(x <= 20, torch.log1p(torch.exp(x.clamp(max=20))), x)


def _per_channel(M, l, gidx):
    """B or C of step l for every (batch, channel): (b, d, n) from a variable (b, g, n, L) or a constant (d, n) operand."""
    return M[:, :, :, l][:, gidx] if M.dim() == 4 else M[None]


def ref_fwd(u, delta, A, B, C, D=None, z=None, bias=None, softplus=False, mutate=None):
    """fp64 selective-scan forward.  u, delta, z: (b, d, L); A (d, n); B, C: (b, g, n, L) or constant (d, n); D, bias: (d,).
    delta' = softplus20(delta + bias);  h_l = exp(delta'_l A) h_{l-1} + delta'_l u_l B_l (h_0 = 0);
    y_l = C_l . h_l + D u_l, times z sigma(z).  Returns y, its magnitude M_y, the states after every step (hs[l] = h after
    l + 1 steps), their error magnitudes Es, and delta'.  mutate (the CPU self-checks only): drop_step l / drop_state n /
    drop_D."""
    mutate = mutate or {}
    b, d, L = u.shape
    n = A.shape[1]
    G = B.shape[1] if B.dim() == 4 else (C.shape[1] if C.dim() == 4 else 1)
    gidx = torch.arange(d, device=u.device) // (d // G)
    dl = delta + (bias[None, :, None] if bias is not None else 0)
    if softplus:
        dl = softplus20(dl)
    h = torch.zeros(b, d, n, dtype=F64, device=u.device)
    E = torch.zeros_like(h)
    ys, Ms, hs, Es = [], [], [], []
    keep = torch.ones(n, dtype=F64, device=u.device)
    if "drop_state" in mutate:
        keep[mutate["drop_state"]] = 0
    for l in range(L):
        dA = dl[:, :, l, None] * A[None]
        a = torch.exp(dA)
        Bl, Cl = _per_channel(B, l, gidx), _per_channel(C, l, gidx)
        x = dl[:, :, l, None] * u[:, :, l, None] * Bl
        if mutate.get("drop_step") == l:
            x = torch.zeros_like(x)
        E = a * E + (1 + dA.abs()) * a * h.abs() + x.abs()
        h = a * h + x
        y = (Cl * h * keep).sum(-1)
        M = (Cl.abs() * (E + h.abs())).sum(-1)
        if D is not None and not mutate.get("drop_D"):
            y = y + D[None] * u[:, :, l]
            M = M + (D[None] * u[:, :, l]).abs()
        ys.append(y)
        Ms.append(M)
        hs.append(h)
        Es.append(E)
    y, M = torch.stack(ys, -1), torch.stack(Ms, -1)
    if z is not None:
        g = z * torch.sigmoid(z)
        y, M = y * g, M * g.abs()
    return dict(y=y, M_y=M, hs=hs, Es=Es, dl=dl)


def ckpt_of(states, L):
    """The checkpoint slots the forward writes: slot k holds the state after min(8 (k + 1), L) steps (scan_fwd.cuh ckpt_after)."""
    return torch.stack([states[min(CK * (k + 1), L) - 1] for k in range((L + CK - 1) // CK)], 1)


def ref_bwd(u, delta, A, B, C, D, z, bias, softplus, dout, mutate=None):
    """fp64 selective-scan backward, the formulas of scan_bwd.cuh's header restated (checked against autograd on the CPU):
        dy_l = dout_l z_l sigma(z_l)                dz_l = dout_l ypre_l sigma(z_l) (1 + z_l (1 - sigma(z_l)))
        dh_l = dy_l C_l + a_{l+1} dh_{l+1}          du_l = dy_l D + delta'_l sum_n dh_l B_l
        dd'_l = sum_n dh_l (h_{l-1} a_l A + B_l u_l)          ddelta_l = dd'_l sigmoid(delta_l + bias) (softplus'; 1 above 20)
        dA = sum_{b,l} dh_l h_{l-1} a_l delta'_l    dD = sum_{b,l} dy_l u_l      dbias = sum_{b,l} ddelta_l
        dB_l = sum_{d in group} dh_l delta'_l u_l   dC_l = sum_{d in group} dy_l h_l   (constant B / C: summed over b and l)
    with magnitudes: G_l = a_{l+1} G_{l+1} + (1 + |delta'_{l+1} A|) a_{l+1} |dh_{l+1}| + |dy_l C_l| for the error of dh,
    the elementwise outputs' M from |dh| + G and the forward's E, and S for the sums.  mutate: drop_dh_step l (dh_l loses the
    a_{l+1} dh_{l+1} term), drop_channel c (the dB / dC sums lose channel c)."""
    mutate = mutate or {}
    f = ref_fwd(u, delta, A, B, C, D, None, bias, softplus)
    b, d, L = u.shape
    n = A.shape[1]
    varB, varC = B.dim() == 4, C.dim() == 4
    G = B.shape[1] if varB else (C.shape[1] if varC else 1)
    gidx = torch.arange(d, device=u.device) // (d // G)
    dl, hs, Es = f["dl"], f["hs"], f["Es"]
    ypre, M_ypre = f["y"], f["M_y"]
    if z is not None:
        sg = torch.sigmoid(z)
        dy, M_dy = dout * z * sg, (dout * z * sg).abs()
        dzf = sg * (1 + z * (1 - sg))
        dz, M_dz = dout * ypre * dzf, (dout * sg * (1 + (z * (1 - sg)).abs())).abs() * M_ypre     # (1 + z (1 - sg) cancels near z = -1.28)
    else:
        dy, M_dy, dz, M_dz = dout, dout.abs(), None, None
    chmask = torch.ones(d, dtype=F64, device=u.device)
    if "drop_channel" in mutate:
        chmask[mutate["drop_channel"]] = 0

    def group_sum(x):           # (b, d, n) -> (b, G, n): sum over the channels of each group
        return x.view(b, G, d // G, n).sum(2)
    zeros = torch.zeros(b, d, n, dtype=F64, device=u.device)
    dh, Gm = zeros.clone(), zeros.clone()
    a_next, dA_next = zeros.clone(), zeros.clone()
    du, M_du, ddl, M_ddl = (torch.zeros(b, d, L, dtype=F64, device=u.device) for _ in range(4))
    dA, S_dA = torch.zeros(d, n, dtype=F64, device=u.device), torch.zeros(d, n, dtype=F64, device=u.device)
    mk = lambda var: torch.zeros(b, G, n, L, dtype=F64, device=u.device) if var else torch.zeros(d, n, dtype=F64, device=u.device)
    dBv, dCv, S_dB, S_dC = mk(varB), mk(varC), mk(varB), mk(varC)
    for l in range(L - 1, -1, -1):
        Bl, Cl = _per_channel(B, l, gidx), _per_channel(C, l, gidx)
        hprev = hs[l - 1] if l > 0 else zeros
        Eprev = Es[l - 1] if l > 0 else zeros
        dAl = dl[:, :, l, None] * A[None]
        a = torch.exp(dAl)
        carry = a_next * dh if mutate.get("drop_dh_step") != l else zeros
        Gm = a_next * Gm + (1 + dA_next.abs()) * a_next * dh.abs() + M_dy[:, :, l, None] * Cl.abs()
        dh = dy[:, :, l, None] * Cl + carry
        Mdh = dh.abs() + Gm
        a_next, dA_next = a, dAl
        dlu = dl[:, :, l, None] * u[:, :, l, None]
        du[:, :, l] = (dh * Bl).sum(-1) * dl[:, :, l] + (dy[:, :, l] * D[None] if D is not None else 0)
        M_du[:, :, l] = (Mdh * Bl.abs()).sum(-1) * dl[:, :, l].abs() + ((dy[:, :, l] * D[None]).abs() if D is not None else 0)
        hm = hprev.abs() + Eprev
        ddl[:, :, l] = (dh * (hprev * a * A[None] + Bl * u[:, :, l, None])).sum(-1)
        M_ddl[:, :, l] = (Mdh * (hm * a * A[None].abs() * (1 + dAl.abs()) + (Bl * u[:, :, l, None]).abs())).sum(-1)
        tA = dh * hprev * a * dl[:, :, l, None]
        dA += tA.sum(0)
        S_dA += (Mdh * hm * a * (1 + dAl.abs()) * dl[:, :, l, None].abs()).sum(0)
        tB, sB = dh * dlu * chmask[None, :, None], Mdh * dlu.abs()
        tC, sC = dy[:, :, l, None] * hs[l] * chmask[None, :, None], M_dy[:, :, l, None] * (hs[l].abs() + Es[l])
        if varB:
            dBv[:, :, :, l], S_dB[:, :, :, l] = group_sum(tB), group_sum(sB)
        else:
            dBv += tB.sum(0)
            S_dB += sB.sum(0)
        if varC:
            dCv[:, :, :, l], S_dC[:, :, :, l] = group_sum(tC), group_sum(sC)
        else:
            dCv += tC.sum(0)
            S_dC += sC.sum(0)
    if softplus:
        pre = delta + (bias[None, :, None] if bias is not None else 0)
        sp = torch.where(pre <= 20, torch.sigmoid(pre), torch.ones_like(pre))
        ddelta, M_ddelta = ddl * sp, M_ddl * sp
    else:
        ddelta, M_ddelta = ddl, M_ddl
    out = dict(du=du, M_du=M_du, ddelta=ddelta, M_ddelta=M_ddelta, dz=dz, M_dz=M_dz, dA=dA, S_dA=S_dA,
               dB=dBv, S_dB=S_dB, dC=dCv, S_dC=S_dC,
               dD=(dy * u).sum((0, 2)), S_dD=(M_dy * u.abs()).sum((0, 2)),
               dbias=ddelta.sum((0, 2)), S_dbias=M_ddelta.sum((0, 2)))
    return out


# ------------------------------------------------------------------------------------------------ CPU: reference and bounds
def _tiny_inputs(b, d, L, n, G, varB, varC, seed, dtype=F64):
    g = torch.Generator().manual_seed(seed)
    rn = lambda *s: torch.randn(*s, generator=g, dtype=F64)
    u, delta, z = rn(b, d, L), 0.5 * rn(b, d, L), rn(b, d, L)
    A = -(0.2 + torch.rand(d, n, generator=g, dtype=F64))
    B = rn(b, G, n, L) if varB else rn(d, n)
    C = rn(b, G, n, L) if varC else rn(d, n)
    D, bias = rn(d), 0.3 * rn(d)
    return [t.to(dtype).to(F64) for t in (u, delta, A, B, C, D, z, bias)]


def test_backward_reference_matches_fp64_autograd():
    """CPU: ref_bwd's explicit formulas equal torch.autograd through ref_fwd, to ~1e-12, for every combination of D, z, bias,
    softplus and variable / constant B and C (two groups where both are variable)."""
    combos = list(itertools.product((False, True), repeat=6))
    for i, (hasD, hasZ, hasBias, sp, varB, varC) in enumerate(combos):
        G = 2 if (varB and varC) else 1
        u, delta, A, B, C, D, z, bias = _tiny_inputs(2, 6, 11, 3, G, varB, varC, seed=i)
        D, z, bias = (D if hasD else None), (z if hasZ else None), (bias if hasBias else None)
        if sp and i % 3 == 0:
            delta[0, 1, 3] = 25.0                         # one element above the softplus threshold
        leaves = [t.clone().requires_grad_() for t in (u, delta, A, B, C)]
        opt = [None if t is None else t.clone().requires_grad_() for t in (D, z, bias)]
        y = ref_fwd(*leaves, opt[0], opt[1], opt[2], sp)["y"]
        dout = torch.randn(y.shape, generator=torch.Generator().manual_seed(99 + i), dtype=F64)
        (y * dout).sum().backward()
        r = ref_bwd(u, delta, A, B, C, D, z, bias, sp, dout)
        want = dict(du=leaves[0].grad, ddelta=leaves[1].grad, dA=leaves[2].grad, dB=leaves[3].grad, dC=leaves[4].grad,
                    dD=opt[0].grad if hasD else None, dz=opt[1].grad if hasZ else None, dbias=opt[2].grad if hasBias else None)
        for k, w in want.items():
            if w is None:
                continue
            got = r[k]
            err = (got - w).abs().max().item() / max(1.0, w.abs().max().item())
            assert err < 1e-12, f"combo {i} (D={hasD} z={hasZ} bias={hasBias} softplus={sp} varB={varB} varC={varC}): {k} off by {err:.2e}"


def _selfcheck_case(T, L=40, d=128, n=8, seed=0):
    u, delta, A, B, C, D, z, bias = _tiny_inputs(2, d, L, n, 1, True, True, seed, dtype=T)
    return u, delta, A, B, C, D, z, bias


@pytest.mark.parametrize("T", DTYPES, ids=[DTYPE_NAME[t] for t in DTYPES])
def test_forward_bounds_reject_dropped_terms(T):
    """CPU: the forward bounds pass the reference rounded to T and reject a forward that drops one step's input term (at l = 0,
    at the chunk boundaries 8 and 16, at L - 1), misses one state or D u, writes its result one position off, or takes a
    checkpoint from the wrong slot."""
    L = 40
    args = _selfcheck_case(T, L)
    r = ref_fwd(*args, softplus=True)
    c = max(C_FAMILY.values())
    check_elem("selfcheck y", r["y"].to(T), r["y"], r["M_y"], c_f32=c)
    ck, M_ck = ckpt_of(r["hs"], L), ckpt_of(r["Es"], L)
    check_elem("selfcheck ckpt", ck.float(), ck, M_ck, c_f32=c)

    def rejects(what, got, e, M):
        with pytest.raises(AssertionError):
            check_elem(what, got, e, M, c_f32=c)
    for mut in [dict(drop_step=l) for l in (0, 8, 16, L - 1)] + [dict(drop_state=3), dict(drop_state=7), dict(drop_D=True)]:
        m = ref_fwd(*args, softplus=True, mutate=mut)
        rejects(f"mutant {mut}", m["y"].to(T), r["y"], r["M_y"])
    rejects("shifted output", torch.roll(r["y"], 1, -1).to(T), r["y"], r["M_y"])
    rejects("wrong slot", torch.roll(ck, 1, 1).float(), ck, M_ck)
    m = ref_fwd(*args, softplus=True, mutate=dict(drop_step=16))
    rejects("ckpt of a forward without step 16", ckpt_of(m["hs"], L).float(), ck, M_ck)


@pytest.mark.parametrize("T", DTYPES, ids=[DTYPE_NAME[t] for t in DTYPES])
def test_backward_bounds_reject_dropped_terms(T):
    """CPU: the backward bounds pass the reference and reject a du missing one step of dh propagation, and dB / dC missing
    one channel of a 64- or 128-channel group."""
    c = max(C_FAMILY.values())
    for d in (64, 128):
        args = _selfcheck_case(T, 24, d, 8, seed=d)
        dout = torch.randn(args[0].shape, generator=torch.Generator().manual_seed(5), dtype=F64).to(T).to(F64)
        r = ref_bwd(*args, True, dout)
        check_elem("selfcheck du", r["du"].to(T), r["du"], r["M_du"], c_f32=c)
        check_colsum("selfcheck dB", r["dB"].float(), r["dB"], r["S_dB"], rel=SUM_REL)
        for l in (0, 7, 8, 15):
            m = ref_bwd(*args, True, dout, mutate=dict(drop_dh_step=l))
            with pytest.raises(AssertionError):
                check_elem(f"du without dh step {l}", m["du"].to(T), r["du"], r["M_du"], c_f32=c)
        for ch in (0, d // 2, d - 1):
            m = ref_bwd(*args, True, dout, mutate=dict(drop_channel=ch))
            for k in ("dB", "dC"):
                with pytest.raises(AssertionError):
                    check_colsum(f"{k} without channel {ch}", m[k].float(), r[k], r["S_" + k], rel=SUM_REL)


# ------------------------------------------------------------------------------------------------ case matrix
class Case(dict):
    """One matrix entry; a flag it does not name reads as None."""
    __getattr__ = dict.get

    def __missing__(self, key):
        return None


def _cases():
    """The matrix.  Each entry names its shape and flags; values rotate with the index so every instantiation meets the edges."""
    out = []
    vals = ("normal", "sp_edge", "sp_neg", "a_edge", "u0_z", "cancel")
    i = 0

    def add(**kw):
        nonlocal i
        kw.setdefault("G", 1)
        kw.setdefault("varB", True)
        kw.setdefault("varC", True)
        kw.setdefault("layout", "tok")
        kw.setdefault("values", vals[i % len(vals)])
        kw.setdefault("hasD", i % 4 != 1)
        kw.setdefault("hasZ", i % 4 != 2)
        kw.setdefault("hasBias", i % 4 != 3)
        kw.setdefault("softplus", i % 5 != 4)
        kw.setdefault("bwd", True)
        if kw["values"] in ("sp_edge", "sp_neg", "long"):
            kw["softplus"] = True
        kw["i"] = i
        out.append(Case(kw))
        i += 1
    # generic forward / backward: every dstate bucket, both layouts, every dtype, constant B / C, groups, ragged shapes
    for T in DTYPES:
        for N, dim, L, G in ((1, 96, 45, 1), (4, 136, 17, 1), (7, 64, 9, 1), (8, 128, 16, 2), (12, 1, 15, 1), (16, 96, 45, 1),
                             (24, 136, 7, 1), (33, 96, 8, 1), (64, 64, 16, 1)):
            for layout in ("chan", "tok"):
                add(T=T, batch=2, dim=dim, L=L, N=N, G=G, layout=layout)
        for N in (4, 16):
            for varB, varC in ((False, True), (True, False), (False, False)):
                add(T=T, batch=2, dim=96, L=45, N=N, layout=("chan", "tok")[(N + varB) % 2], varB=varB, varC=varC)
        # constant B / C beyond dstate 16: no forward kernel; the backward runs from the reference's checkpoints
        for N in (24, 64):
            add(T=T, batch=2, dim=64, L=17, N=N, layout="chan", varB=False, varC=True, fwd=False)
        add(T=T, batch=2, dim=3 * 84, L=16, N=16, G=3, layout="tok")                          # 84 channels per group: ragged tiles
        add(T=T, batch=2, dim=4 * 80, L=9, N=8, G=4, layout="chan")
        add(T=T, batch=2, dim=64, L=1, N=16, layout="tok")
        add(T=T, batch=2, dim=64, L=277, N=16, layout="chan", values="a_edge")
        add(T=T, batch=65537, dim=64, L=8, N=1, layout="chan", values="normal")              # 1-D grid above 65535
        add(T=T, batch=2, dim=64, L=1024, N=16, layout="tok", values="long")
        add(T=T, batch=1, dim=64, L=4096, N=8, layout="chan", values="long")
        add(T=T, batch=2, dim=128, L=64, N=16, layout="tok", sliced=True)                     # B / C as column views of x_dbl rows
    # hot path (16-bit, token-major, dstate 16): the CTA-wide kernel, its fallbacks, the fused options
    for T in LOWP:
        for dim, L, G in ((128, 64, 1), (64, 8, 1), (256, 40, 2), (192, 264, 1), (128, 16, 1)):
            add(T=T, batch=2, dim=dim, L=L, N=16, G=G, sliced=True)
            add(T=T, batch=2, dim=dim, L=L, N=16, G=G, sliced=True, rowmap=True, hasZ=True, values="normal")
        add(T=T, batch=2, dim=128, L=64, N=16, sliced=True, rowmap=True, hasZ=True, hasD=True, softplus=True, hasBias=True, values="normal")
        add(T=T, batch=65537, dim=64, L=8, N=16, sliced=True, values="normal", hasZ=True, softplus=True)   # 1-D grid, hot path
        for what in ("D", "A", "bias"):              # misaligned D / A / delta_bias: the tpc2 kernel (L % 16 == 0) or generic
            add(T=T, batch=2, dim=128, L=64, N=16, sliced=True, misalign=what, hasD=True, hasBias=True)
            add(T=T, batch=2, dim=128, L=40, N=16, sliced=True, misalign=what, hasD=True, hasBias=True)
        add(T=T, batch=2, dim=128, L=48, N=16, layout="chan", misalign="Acontig")             # A 4 bytes off 16: the generic bwd
        add(T=T, batch=2, dim=128, L=48, N=16, layout="chan", strided=True)                   # strides that force q4 unstaged
        add(T=T, batch=2, dim=96, L=45, N=16, layout="tok", strided=True)
        add(T=T, batch=2, dim=128, L=64, N=16, sliced=True, rowmap=True, hasZ=True, reverse=True, bwd=False)
        add(T=T, batch=2, dim=128, L=64, N=16, sliced=True, rowmap=True, hasZ=True, reverse=True, accumulate=True, bwd=False)
        add(T=T, batch=2, dim=128, L=64, N=16, sliced=True, hasZ=False, reverse=True, accumulate=True, bwd=False)
        add(T=T, batch=8, dim=128, L=16, N=16, rowmap=True, hasZ=True, btk=4, bwd=False)      # two-level z batch (video)
        for R in (40, 48):
            add(T=T, batch=2, dim=128, L=64, N=16, dt_rank=R, rowmap=True, hasZ=True, softplus=True, bwd=False)
            add(T=T, batch=2, dim=192, L=24, N=16, dt_rank=R, hasZ=False, softplus=True, bwd=False)
        for batch, dim, mode in ((64, 1280, 3), (40, 1280, 5), (8, 1280, 0)):                  # scan_kernel_choice at 132 SMs
            add(T=T, batch=batch, dim=dim, L=16, N=16, sliced=True, auto_mode=mode, hasZ=True, softplus=True, values="normal")
            add(T=T, batch=batch, dim=dim, L=8, N=16, sliced=True, auto_mode=mode, hasZ=False, values="normal", bwd=False)
    return out


CASES = _cases()


def _case_id(c):
    s = f"{c.i}-{DTYPE_NAME[c.T]}-b{c.batch}-d{c.dim}-L{c.L}-N{c.N}-{c.layout}"
    for k in ("sliced", "rowmap", "reverse", "accumulate", "strided"):
        if c[k]:
            s += f"-{k}"
    for k in ("misalign", "dt_rank", "btk", "auto_mode"):
        if c[k] is not None:
            s += f"-{k}{c[k]}"
    if not (c.varB and c.varC):
        s += f"-const{'B' if not c.varB else ''}{'C' if not c.varC else ''}"
    return s + f"-{c['values']}"


def make_inputs(c):
    """Inputs of one case, drawn in the kernel dtype on the CPU (u, delta, z, B, C in T; A, D, bias, constant B / C fp32)."""
    g = torch.Generator().manual_seed(7919 * c.i + 13)
    rn = lambda *s: torch.randn(*s, generator=g)
    ru = lambda *s: torch.rand(*s, generator=g)
    b, d, L, n, G = c.batch, c.dim, c.L, c.N, c.G
    T = c.T
    u, z = rn(b, d, L), rn(b, d, L)
    # delta' >= 0 without softplus (a <= 1, as in every model); with it, delta + bias may be negative
    delta = 0.5 * ru(b, d, L) - (0.1 if c.softplus else 0.0)
    A = -(0.1 + ru(d, n))
    Bv = rn(b, G, n, L) if c.varB else rn(d, n)
    Cv = rn(b, G, n, L) if c.varC else rn(d, n)
    D, bias = rn(d), (0.3 * rn(d) if c.softplus else 0.3 * ru(d))
    v = c["values"]
    if v == "sp_edge":              # delta + bias across the softplus threshold (delta 0 in T, the edge in the fp32 bias)
        for k, x in enumerate((19.99, 20.0, 20.01)):
            if k < d:
                delta[:, k], bias[k] = 0.0, x
        A[: min(3, d)] *= 0.01
    elif v == "sp_neg":             # the log1p series branch, and e^-100 flushed to zero by ex2.approx.ftz
        for k, x in enumerate((-30.0, -100.0)):
            if k < d:
                delta[:, k], bias[k] = 0.0, x
    elif v == "a_edge":             # a == 1, and a that underflows
        A[0] = 0.0
        if d > 1:
            A[1] = -1e4
            delta[:, 1] += 1.0
    elif v == "u0_z":               # u == 0 rows; z at +-30 and near 0
        u[:, 0] = 0.0
        if d > 3:
            z[:, 1], z[:, 2], z[:, 3] = 30.0, -30.0, 1e-3 * z[:, 3]
    elif v == "cancel" and n >= 2:  # paired states with opposite C: large |u B| that cancels in y
        m = n // 2 * 2
        A[:, 1:m:2] = A[:, 0:m:2]
        if c.varB:
            Bv[:, :, 1:m:2] = Bv[:, :, 0:m:2]
        else:
            Bv[:, 1:m:2] = Bv[:, 0:m:2]
        if c.varC:
            Cv[:, :, 1:m:2] = -Cv[:, :, 0:m:2]
        else:
            Cv[:, 1:m:2] = -Cv[:, 0:m:2]
        u *= 100.0
    elif v == "long":               # long accumulation: A near 0, small steps
        A = -1e-3 * ru(d, n)
        delta = 0.05 * ru(b, d, L)
        bias = torch.zeros(d) - 3.0
    dout = rn(b, d, L)
    x = dict(u=u.to(T), delta=delta.to(T), z=z.to(T), A=A, D=D, bias=bias, dout=dout.to(T),
             B=Bv.to(T) if c.varB else Bv, C=Cv.to(T) if c.varC else Cv)
    if c.dt_rank:
        R = c.dt_rank
        # dyadic rationals: the fp32 tensor-core sums are exact in any order, so delta rounds as in the fp64 reference
        x["xdt"] = (torch.randint(-16, 17, (b, L, R), generator=g) / 8).to(T)
        x["wdt"] = (torch.randint(-8, 9, (d, R), generator=g) / 64).to(T)
    if c.accumulate:
        x["P"] = rn(b, L, d).to(T)
    if c.btk:
        K = c.btk
        x["zfull"] = rn(b // K, L, K, 2 * d).to(T)
    return x


def _tok(t):
    """(b, d, L) logical view of a token-major (b, L, d) copy."""
    return t.transpose(1, 2).contiguous().transpose(1, 2)


def _misaligned(t, elems):
    """A copy of t that starts `elems` elements past an allocation: contiguous, but only 4-byte aligned."""
    buf = torch.empty(t.numel() + elems, dtype=t.dtype, device=DEV)
    v = buf[elems:].view(t.shape)
    v.copy_(t)
    return v


def device_args(c, x):
    """The kernel call's tensors, in the case's layout (token-major, channel-first, sliced, strided, misaligned)."""
    T = c.T
    b, d, L, n = c.batch, c.dim, c.L, c.N
    u, delta, z = (x[k].to(DEV) for k in ("u", "delta", "z"))
    if c.layout == "tok":
        u, delta, z = _tok(u), _tok(delta), _tok(z)
    if c.strided:               # rows with a stride that is not a whole number of 16-byte chunks
        def pad(t):
            wide = torch.zeros(b, d, L + 3, dtype=T, device=DEV) if c.layout == "chan" else torch.zeros(b, L, d + 1, dtype=T, device=DEV).transpose(1, 2)
            wide[:, :d, :L] = t
            return wide[:, :d, :L]
        u, delta, z = pad(u), pad(delta), pad(z)
    B, C = x["B"].to(DEV), x["C"].to(DEV)
    if c.sliced and c.varB and c.varC and c.layout == "tok" and not c.dt_rank:
        # B and C as views of x_dbl rows (b, L, R + 2 G n): the model's layout, R = 8 delta-rank columns ahead of them
        R = 8
        xdbl = torch.zeros(b, L, R + 2 * c.G * n, dtype=T, device=DEV)
        xdbl[:, :, R:R + c.G * n] = B.permute(0, 3, 1, 2).reshape(b, L, c.G * n)
        xdbl[:, :, R + c.G * n:] = C.permute(0, 3, 1, 2).reshape(b, L, c.G * n)
        B = xdbl[:, :, R:R + c.G * n].view(b, L, c.G, n).permute(0, 2, 3, 1)
        C = xdbl[:, :, R + c.G * n:].view(b, L, c.G, n).permute(0, 2, 3, 1)
    elif c.layout == "tok":
        if c.varB:
            B = B.transpose(2, 3).contiguous().transpose(2, 3)
        if c.varC:
            C = C.transpose(2, 3).contiguous().transpose(2, 3)
    A, D, bias = x["A"].to(DEV), x["D"].to(DEV), x["bias"].to(DEV)
    if c.misalign == "Acontig":
        A = _misaligned(A, 1)
    elif c.misalign in ("A", "D", "bias"):      # a view 4 bytes past an 8-byte boundary
        if c.misalign == "A":
            A = _misaligned(A, 1)
        elif c.misalign == "D":
            D = _misaligned(D, 1)
        else:
            bias = _misaligned(bias, 1)
    dt = None
    if c.dt_rank:
        R = c.dt_rank
        xdbl = torch.cat([x["xdt"], x["B"][:, 0].permute(0, 2, 1), x["C"][:, 0].permute(0, 2, 1)], 2).to(DEV)
        B = xdbl[:, :, R:R + n].permute(0, 2, 1).unsqueeze(1)
        C = xdbl[:, :, R + n:].permute(0, 2, 1).unsqueeze(1)
        dt = (x["wdt"].to(DEV), xdbl)
        delta = None
    return dict(u=u, delta=delta, z=z if c.hasZ else None, A=A, B=B, C=C, D=D if c.hasD else None,
                bias=bias if c.hasBias else None, dt=dt)


def _rowmap(c):
    return torch.randperm(c.L, generator=torch.Generator().manual_seed(c.i)).to(torch.int32)


def reference_inputs(c, x):
    """fp64 (on the GPU) operands of the reference, with the hot-path options folded in: the rounded dt_proj product as delta,
    the gathered z."""
    dv = lambda t: t.to(DEV).to(F64)
    u, delta, z = dv(x["u"]), dv(x["delta"]) if not c.dt_rank else None, dv(x["z"])
    if c.dt_rank:
        # delta = round_T(W_dt . x_dbl[:, :R]) (the kernel rounds the tensor-core product like the reference's GEMM output)
        delta = torch.einsum("blr,er->bel", dv(x["xdt"]), dv(x["wdt"])).to(c.T).to(F64)
    if c.rowmap:
        perm = _rowmap(c).long().to(DEV)
        if c.btk:
            K = c.btk
            zf = dv(x["zfull"])[..., c.dim:]                      # (B, L, K, d)
            z = zf[:, perm].permute(0, 2, 3, 1).reshape(c.batch, c.dim, c.L)
        else:
            z = z[:, :, perm]
    B = dv(x["B"]) if c.varB else x["B"].to(DEV).to(F64)
    C = dv(x["C"]) if c.varC else x["C"].to(DEV).to(F64)
    return [u, delta, x["A"].to(DEV).to(F64), B, C, x["D"].to(DEV).to(F64) if c.hasD else None,
            z if c.hasZ or c.btk else None, x["bias"].to(DEV).to(F64) if c.hasBias else None]


# ------------------------------------------------------------------------------------------------ running the kernels
def _fwd_family(name):
    for key, fam in (("wp", "fwd_wp"), ("tpc2", "fwd_tpc2"), ("tma", "fwd_tma")):
        if f"scan_fwd_{key}" in name:
            return fam
    return "fwd_generic"


def run_fwd(c, x, args, want_ckpt):
    from zigma_b200 import _lib
    from zigma_b200.selective_scan_interface import _scan_fwd
    kw = dict(want_last_state=not (c.reverse or c.accumulate), want_ckpt=want_ckpt)
    z = args["z"]
    if c.rowmap:
        kw["z_rowmap"] = _rowmap(c).to(DEV)
    if c.btk:
        zf = x["zfull"].to(DEV)
        kw["z_btk"] = zf[..., c.dim:]
        z = None
    if c.dt_rank:
        kw["dt_proj"] = args["dt"]
    out_buf = None
    if c.reverse:
        out_buf = x["P"].to(DEV).clone() if c.accumulate else torch.empty(c.batch, c.L, c.dim, dtype=c.T, device=DEV)
        kw.update(out=out_buf.transpose(1, 2), out_reverse=True, out_accumulate=bool(c.accumulate))
    y, last, ck, saved = _scan_fwd(args["u"], args["delta"], args["A"], args["B"], args["C"], args["D"], z, args["bias"],
                                   c.softplus, **kw)
    return dict(y=y, last=last, ckpt=ck, saved=saved, kernel=_lib.last_scan_kernel(), buf=out_buf)


def check_fwd(tag, c, r, got, Ls=None):
    fam = _fwd_family(got["kernel"])
    cf = C_FAMILY[fam]
    tag = f"{fam} {tag}"
    e, M = r["y"], r["M_y"]
    if c.reverse:
        e, M = e.flip(-1), M.flip(-1)
        y = got["buf"].transpose(1, 2)
        if c.accumulate:
            P = c["_P"]
            ey = e
            e, M = P + ey.to(c.T).to(F64), P.abs() + M
            check_elem(f"{tag} y (reverse, accumulate)", y, e, M, max_ulp=2, extra=ulp(ey, c.T), c_f32=cf, mismatch=MISMATCH.get(c.T), conditioned=True)
            return
        check_elem(f"{tag} y (reverse)", y, e, M, c_f32=cf, mismatch=MISMATCH.get(c.T), conditioned=True)
        return
    check_elem(f"{tag} y", got["y"], e, M, c_f32=cf, mismatch=MISMATCH.get(c.T), conditioned=True)
    if got["last"] is not None:
        check_elem(f"{tag} last_state", got["last"], r["hs"][-1], r["Es"][-1], c_f32=cf)
    if got["ckpt"] is not None:
        check_elem(f"{tag} ckpt (every slot)", got["ckpt"], ckpt_of(r["hs"], c.L), ckpt_of(r["Es"], c.L), c_f32=cf)


def _bwd_family(c, args):
    q4 = c.N == 16 and c.varB and c.varC and args["A"].data_ptr() % 16 == 0
    return "bwd_q4" if q4 else "bwd_generic"


def run_bwd(c, x, args, saved, ckpt, det):
    from zigma_b200.selective_scan_interface import _scan_bwd
    dout = x["dout"].to(DEV)
    if c.layout == "tok":
        dout = _tok(dout)
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(det)
    try:
        kw = dict(z_rowmap=_rowmap(c).to(DEV)) if c.rowmap else {}
        return _scan_bwd(saved, ckpt, dout, c.softplus, **kw)
    finally:
        torch.use_deterministic_algorithms(prev)


def check_bwd(tag, c, rb, got, fam):
    du, ddelta, dA, dB, dC, dD, dbias, dz = got
    cf = C_FAMILY[fam]
    tag = f"{fam} {tag}"
    check_elem(f"{tag} du", du, rb["du"], rb["M_du"], c_f32=cf, mismatch=MISMATCH.get(c.T), conditioned=True)
    check_elem(f"{tag} ddelta", ddelta, rb["ddelta"], rb["M_ddelta"], c_f32=cf, mismatch=MISMATCH.get(c.T), conditioned=True)
    if c.hasZ:
        dzv = dz
        if c.rowmap:                                  # dz written in token order: scan step l lands on row rowmap[l]
            perm = _rowmap(c).long().to(DEV)
            dzv = dz[:, :, perm]
        check_elem(f"{tag} dz", dzv, rb["dz"], rb["M_dz"], c_f32=cf, mismatch=MISMATCH.get(c.T), conditioned=True)
    check_colsum(f"{tag} dA", dA, rb["dA"], rb["S_dA"], rel=SUM_REL)
    check_colsum(f"{tag} dB", dB if c.varB else dB, rb["dB"], rb["S_dB"], rel=SUM_REL)
    check_colsum(f"{tag} dC", dC, rb["dC"], rb["S_dC"], rel=SUM_REL)
    if c.hasD:
        check_colsum(f"{tag} dD", dD, rb["dD"], rb["S_dD"], rel=SUM_REL)
    if c.hasBias:
        check_colsum(f"{tag} dbias", dbias, rb["dbias"], rb["S_dbias"], rel=SUM_REL)


def run_case(c, check=True, dets=(False, True)):
    """Forward (the training call with checkpoints and the inference call without; one of them where the options allow only
    one), then the backward from the training call's checkpoints, with and without the deterministic flag, each against the
    fp64 references (computed on the GPU).  Returns the names of the forward kernels that ran."""
    from zigma_b200 import _lib
    x = make_inputs(c)
    args = device_args(c, x)
    kernels = []
    ref_in = reference_inputs(c, x) if check else None
    if c.accumulate:
        c["_P"] = x["P"].to(DEV).to(F64).transpose(1, 2)
    saved = ckpt = None
    if c.fwd is not False:
        r = ref_fwd(*ref_in, softplus=c.softplus) if check else None
        calls = (False,) if (c.reverse or c.btk) else (True, False)
        for want_ckpt in calls:
            got = run_fwd(c, x, args, want_ckpt)
            kernels.append(got["kernel"])
            if c.auto_mode is not None and not want_ckpt:
                mode = _lib.scan_kernel_choice(c.batch, c.dim, sms=132)[0]
                assert mode == c.auto_mode, (mode, c.auto_mode)
                if torch.cuda.get_device_properties(0).multi_processor_count == 132 and "ZG_SCAN_WP" not in os.environ:
                    want = {0: "scan_fwd_tma_kernel", 3: "scan_fwd_wp2_kernel", 5: "scan_fwd_wph_kernel"}[mode]
                    assert want in got["kernel"], got["kernel"]
            if check:
                check_fwd(f"{_case_id(c)} ckpt={want_ckpt}", c, r, got)
            if want_ckpt:
                saved, ckpt = got["saved"], got["ckpt"]
        del r
    if not c.bwd:
        return kernels
    if c.fwd is False:                  # no forward kernel for this flag set: the backward reads the reference's checkpoints
        r0 = ref_fwd(*reference_inputs(c, x), softplus=c.softplus)
        ckpt = ckpt_of(r0["hs"], c.L).float().contiguous()
        del r0
        saved = (args["u"], args["delta"], args["z"], args["B"].contiguous(), args["C"].contiguous(), args["D"], args["bias"],
                 args["A"].contiguous())
    fam = _bwd_family(c, args)
    rb = ref_bwd(*ref_in, c.softplus, x["dout"].to(DEV).to(F64)) if check else None
    for det in dets:
        got = run_bwd(c, x, args, saved, ckpt, det)
        if check:
            check_bwd(f"{_case_id(c)} det={det}", c, rb, got, fam)
    return kernels


@gpu
@pytest.mark.parametrize("c", CASES, ids=[_case_id(c) for c in CASES])
def test_scan_vs_fp64(c):
    run_case(c)


def _named_case(T, **kw):
    base = dict(T=T, batch=2, dim=64, L=16, N=16, G=1, varB=True, varC=True, layout="tok", values="normal", hasD=True, hasZ=True,
                hasBias=True, softplus=True, bwd=True, i=5000)
    base.update(kw)
    return Case(base)


@gpu
@pytest.mark.parametrize("N", (16, 8), ids=("q4", "generic"))
@pytest.mark.parametrize("T", DTYPES, ids=[DTYPE_NAME[t] for t in DTYPES])
def test_softplus_gradient_far_below_zero(T, N):
    """delta + bias = -30 (and -100): softplus' = sigmoid(-30) = 9.4e-14.  Both backward kernels used to form it as
    1 - exp(-softplus(x)), which is 0 in fp32 there, so ddelta and d(delta_bias) of such channels came out as exact zeros
    (fp32 ddelta off by 3e6 x the bound, fp16 d(delta_bias) by 1.5e4 x).  zg_softplus_grad takes the series below 1/8."""
    run_case(_named_case(T, N=N, values="sp_neg", i=5000 + N))


@gpu
@pytest.mark.parametrize("T", DTYPES, ids=[DTYPE_NAME[t] for t in DTYPES])
def test_backward_with_contiguous_misaligned_A(T):
    """A contiguous A 4 bytes past a 16-byte boundary: the dstate-16 backward cannot take it (16-byte loads), and _scan_bwd used
    to keep the token-major layout anyway, so the generic kernel raised 'needs seq-contiguous tensors'."""
    run_case(_named_case(T, dim=128, L=48, misalign="Acontig", i=5100))


# ------------------------------------------------------------------------------------------------ inventory
def _b(v):
    return "true" if v else "false"


T_ALL = ("float", "__half", "__nv_bfloat16")
T_16 = ("__half", "__nv_bfloat16")


def _inventory():
    """(kernel, template args) of every scan kernel of the library, from the dispatch code of scan_fwd*.cuh / scan_bwd*.cuh: each
    one is reached by some call's inputs alone."""
    dflt = set()
    for t in T_ALL:                                    # generic forward: NS 8 / 16 / 32 / 64, both layouts; constant B / C <= 16
        for ns in (8, 16, 32, 64):
            for seq in (True, False):
                dflt.add(("scan_fwd_kernel", (t, str(ns), _b(seq), "false")))
        for ns in (8, 16):
            for seq in (True, False):
                dflt.add(("scan_fwd_kernel", (t, str(ns), _b(seq), "true")))
    for t in T_16:
        # hot path: R 0 (plain = the model's call: z, softplus, no reverse / accumulate) and the fused dt_proj prologue R 40 / 48
        for ck in (True, False):
            for plain in (False, True):
                dflt.add(("scan_fwd_tma_kernel", (t, "0", _b(ck), _b(plain))))
            for R in ("40", "48"):
                dflt.add(("scan_fwd_tma_kernel", (t, R, _b(ck), "false")))
            dflt.add(("scan_fwd_tpc2_kernel", (t, _b(ck))))               # tpc2 (round-1 fallback)
        for plain in (False, True):                    # inference calls only: wp2 = the automatic choice's mode 3, wph = mode 5
            dflt.add(("scan_fwd_wp2_kernel", (t, _b(plain))))
            dflt.add(("scan_fwd_wph_kernel", (t, _b(plain))))
    for t in T_ALL:                                    # backward: generic (NS, constant B / C), q4 (staged or not), DET both ways
        for det in (False, True):
            for ns in (8, 16, 32, 64):
                for cb in (False, True):
                    dflt.add(("scan_bwd_kernel", (t, str(ns), _b(cb), _b(det))))
            for st in (False, True):
                dflt.add(("scan_bwd_q4_kernel", (t, _b(st), _b(det))))
    return dflt


DEFAULT = _inventory()
SCAN_RE = re.compile(r"zg::(scan_(?:fwd|bwd)\w*_kernel)<(.*)>\(")


def _template_args(s):
    out = []
    for a in s.split(","):
        a = a.strip()
        a = {"(bool)1": "true", "(bool)0": "false"}.get(a, a)
        out.append(re.sub(r"^\((?:int|unsigned int)\)", "", a))
    return tuple(out)


def _tool(name):
    p = os.path.join("/usr/local/cuda/bin", name)
    return shutil.which(name) or (p if os.path.exists(p) else None)


def test_inventory_matches_library():
    """CPU: the zg::scan_fwd* / zg::scan_bwd* kernels in the built library are exactly DEFAULT (124): a new instantiation fails
    here until this file tests it."""
    assert len(DEFAULT) == 124
    cuobjdump, filt = _tool("cuobjdump"), _tool("cu++filt")
    if cuobjdump is None or filt is None:
        pytest.skip("cuobjdump / cu++filt not available")
    import __graft_entry__
    __graft_entry__.build()
    from zigma_b200 import _lib
    listing = subprocess.run([cuobjdump, "-elf", _lib.LIB_PATH], check=True, capture_output=True, text=True).stdout
    names = sorted(set(re.findall(r"\.text\.(_Z\S+)", listing)))
    demangled = subprocess.run([filt], input="\n".join(names), check=True, capture_output=True, text=True).stdout.splitlines()
    found = set()
    for dem in demangled:
        m = SCAN_RE.search(dem)
        if m:
            found.add((m.group(1), _template_args(m.group(2))))
    missing, extra = sorted(DEFAULT - found), sorted(found - DEFAULT)
    assert not missing and not extra, f"in the table, not in the library: {missing}\nin the library, not in the table: {extra}"


def _launched(fn):
    """The scan kernels (name, template args) that fn launches, from torch.profiler."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    seen = set()
    for evt in prof.events():
        m = SCAN_RE.search(evt.name)
        if m:
            seen.add((m.group(1), _template_args(m.group(2))))
    return seen


@gpu
def test_matrix_launches_exactly_default():
    """The matrix, run once more without the references under torch.profiler, launches exactly DEFAULT (64 forward, 60
    backward instantiations)."""
    seen = _launched(lambda: [run_case(c, check=False) for c in CASES])
    missing, extra = sorted(DEFAULT - seen), sorted(seen - DEFAULT)
    assert not missing and not extra, f"not launched: {missing}\nlaunched but not DEFAULT: {extra}"
