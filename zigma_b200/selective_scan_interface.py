"""Host-side mirror of the reference's selective-scan op surface over the sm_90a kernels.

Same names, argument meaning and error behaviour as
``dis_mamba/mamba_ssm/ops/selective_scan_interface.py`` (reference):
``selective_scan_fn`` (:77-83), ``mamba_inner_fn`` (:606-614), ``mamba_inner_fn_no_out_proj``
(:627-633), ``bimamba_inner_fn`` (:616-624).  The arithmetic runs in ``libzigma_b200.so`` through
the C-ABI of ``include/zigma_b200.h``; GEMMs that the reference leaves to cuBLAS (``F.linear`` /
``@``) stay library GEMMs on this autograd path (the inference fast path in ``engine.py`` uses the
fused kernels instead).  No CPU / eager fallback exists: without the native library a
RuntimeError is raised.

Besides the reference surface, ``MambaInnerTokFn`` / ``mamba_inner_tok_fn`` is the token-major training
core that ``Mamba.forward`` uses (same math as ``MambaInnerFnNoOutProj`` on the permuted sequence; the
permutation is folded into the conv / scan kernels in both directions).
"""
import torch
import torch.nn.functional as F

from . import _lib
from .causal_conv1d_interface import _conv_fwd, _conv_bwd

CKPT_EVERY = 8  # recompute-seed spacing: the backward kernel re-runs 8-step chunks from these states


def _strides3(t):
    return t.stride(0), t.stride(1), t.stride(2)


def _scan_fwd(u, delta, A, B, C, D=None, z=None, delta_bias=None, delta_softplus=False,
              z_rowmap=None, want_last_state=True, want_ckpt=False, out=None, dt_proj=None, out_reverse=False, out_accumulate=False, z_btk=None):
    """Raw forward.  u, delta, z: logical (batch, dim, seqlen) tensors (either memory layout, see
    include/zigma_b200.h); B, C: (batch, groups, dstate, seqlen) variable or (dim, dstate) fp32.
    Returns (out, last_state | None, ckpt | None).  Mirrors the checks of selective_scan.cpp:238-300.

    dt_proj = (dt_weight (dim, R), x_dbl (batch, seqlen, >= R + 2 dstate)) with delta=None: the fused dt_proj prologue --
    delta = dt_weight @ x_dbl[..., :R] is formed inside the kernel (tensor cores), B and C must be the views
    x_dbl[..., R:R+N] / x_dbl[..., R+N:R+2N] of the same rows (selective_scan_interface.py:323 of the reference).

    z_btk (instead of z, hot-path kernel only, needs z_rowmap): a (B, T, K, dim) strided view; sequence b' = b K + k of the call
    gates with z_btk[b, :, k, :] -- the factorised temporal scan reading the (b, t k) token-major xz tensor in place.

    out_reverse / out_accumulate (hot-path kernel only, needs ``out``): write step l to position seqlen-1-l / add into ``out``
    with the rounding of an eager 16-bit ``a + b`` -- the second sweep of scan_type "v2" (mamba_simple.py:304-339)."""
    _lib.require_cuda(u, delta, A, B, C, D, z, delta_bias)
    if u.dim() != 3:
        raise RuntimeError("selective_scan: u must be (batch, dim, seqlen)")
    batch, dim, seqlen = u.shape
    if A.is_complex():
        raise NotImplementedError("zigma_b200: complex A is not supported (ZigMa never uses it)")
    dstate = A.shape[1]
    if dt_proj is not None:
        if delta is not None:
            raise RuntimeError("selective_scan: pass either delta or dt_proj, not both")
        dt_w, dt_x = dt_proj
        _lib.require_cuda(dt_w, dt_x)
        if dt_w.dim() != 2 or dt_w.shape[0] != dim or dt_w.dtype != u.dtype or dt_w.stride(1) != 1:
            raise RuntimeError("selective_scan: dt_proj weight must be (dim, dt_rank) in the dtype of u, rows contiguous")
        if dt_x.dim() != 3 or dt_x.shape[0] != batch or dt_x.shape[1] != seqlen or dt_x.dtype != u.dtype or dt_x.stride(2) != 1:
            raise RuntimeError("selective_scan: dt_proj input must be (batch, seqlen, >= dt_rank) rows in the dtype of u")
    elif delta.shape != u.shape or delta.dtype != u.dtype:
        raise RuntimeError("selective_scan: delta must match u in shape and dtype")
    if A.shape != (dim, dstate) or A.dtype != torch.float32:
        raise RuntimeError("selective_scan: A must be fp32 (dim, dstate)")
    A = A.contiguous()
    var_b, var_c = B.dim() >= 3, C.dim() >= 3
    flags = (_lib.SCAN_DELTA_SOFTPLUS if delta_softplus else 0) | (_lib.SCAN_VARIABLE_B if var_b else 0) | (_lib.SCAN_VARIABLE_C if var_c else 0)
    flags |= (_lib.SCAN_OUT_REVERSE if out_reverse else 0) | (_lib.SCAN_OUT_ACCUMULATE if out_accumulate else 0)
    if out_accumulate and out is None:
        raise RuntimeError("selective_scan: out_accumulate needs an existing `out`")
    ngroups = 1
    for name, M, var in (("B", B, var_b), ("C", C, var_c)):
        if var:
            if M.dim() != 4 or M.shape[0] != batch or M.shape[2] != dstate or M.shape[3] != seqlen:
                raise RuntimeError(f"selective_scan: variable {name} must be (batch, groups, dstate, seqlen)")
            if M.dtype != u.dtype:
                raise RuntimeError(f"selective_scan: variable {name} must have the dtype of u")
            ngroups = M.shape[1]
        elif M.shape != (dim, dstate) or M.dtype != torch.float32:
            raise RuntimeError(f"selective_scan: constant {name} must be fp32 (dim, dstate)")
    if var_b and var_c and B.shape[1] != C.shape[1]:
        raise RuntimeError("selective_scan: B and C must have the same number of groups")
    if dim % ngroups != 0:
        raise RuntimeError("selective_scan: dim must be divisible by the number of groups")
    for name, v in (("D", D), ("delta_bias", delta_bias)):
        if v is not None and (v.shape != (dim,) or v.dtype != torch.float32):
            raise RuntimeError(f"selective_scan: {name} must be fp32 (dim,)")
    if z is not None and (z.shape != u.shape or z.dtype != u.dtype):
        raise RuntimeError("selective_scan: z must match u in shape and dtype")
    if z_btk is not None:
        if z is not None or z_rowmap is None:
            raise RuntimeError("selective_scan: z_btk replaces z and needs a z_rowmap")
        Bz, Tz, Kz, Ez = z_btk.shape
        if Bz * Kz != batch or Tz != seqlen or Ez != dim or z_btk.dtype != u.dtype or z_btk.stride(3) != 1:
            raise RuntimeError("selective_scan: z_btk must be (B, seqlen, K, dim) with B * K == batch, dim contiguous")

    seq_layout = u.stride(2) == 1 or seqlen == 1
    if not seq_layout and not (u.stride(1) == 1 or dim == 1):
        u = u.contiguous()
        seq_layout = True
    if out is None:
        if seq_layout:
            out = torch.empty((batch, dim, seqlen), dtype=u.dtype, device=u.device)
        else:   # token-major result, returned as a logical (batch, dim, seqlen) view
            out = torch.empty((batch, seqlen, dim), dtype=u.dtype, device=u.device).transpose(1, 2)

    def fix(t):   # bring an activation into the layout class of u
        if t is None:
            return None
        ok = (t.stride(2) == 1 or seqlen == 1) if seq_layout else (t.stride(1) == 1 or dim == 1)
        if ok:
            return t
        return t.contiguous() if seq_layout else t.transpose(1, 2).contiguous().transpose(1, 2)
    delta, z = fix(delta), fix(z)
    if var_b and not ((B.stride(3) == 1 or seqlen == 1) if seq_layout else (B.stride(2) == 1 or dstate == 1)):
        B = B.contiguous() if seq_layout else B.transpose(2, 3).contiguous().transpose(2, 3)
    if var_c and not ((C.stride(3) == 1 or seqlen == 1) if seq_layout else (C.stride(2) == 1 or dstate == 1)):
        C = C.contiguous() if seq_layout else C.transpose(2, 3).contiguous().transpose(2, 3)
    if not var_b:
        B = B.contiguous()
    if not var_c:
        C = C.contiguous()
    if D is not None:
        D = D.contiguous()
    if delta_bias is not None:
        delta_bias = delta_bias.contiguous()
    if z_rowmap is not None:
        if seq_layout:
            raise RuntimeError("selective_scan: z_rowmap needs token-major (dim-contiguous) activations")
        if z_rowmap.dtype != torch.int32 or z_rowmap.numel() != seqlen or not z_rowmap.is_contiguous():
            raise RuntimeError("selective_scan: z_rowmap must be a contiguous int32 (seqlen,) tensor")

    last = torch.empty((batch, dim, dstate), dtype=torch.float32, device=u.device) if want_last_state else None
    ckpt = None
    if want_ckpt:
        nck = max(1, (seqlen + CKPT_EVERY - 1) // CKPT_EVERY)
        ckpt = torch.empty((batch, nck, dim, dstate), dtype=torch.float32, device=u.device)

    p = _lib.ScanParams()
    p.u, p.delta, p.z, p.B, p.C = _lib.ptr(u), _lib.ptr(delta), _lib.ptr(z), _lib.ptr(B), _lib.ptr(C)
    p.A, p.D, p.delta_bias, p.z_rowmap = _lib.ptr(A), _lib.ptr(D), _lib.ptr(delta_bias), _lib.ptr(z_rowmap)
    p.out, p.last_state, p.ckpt = _lib.ptr(out), _lib.ptr(last), _lib.ptr(ckpt)
    p.u_sb, p.u_sd, p.u_sl = _strides3(u)
    if delta is not None:
        p.delta_sb, p.delta_sd, p.delta_sl = _strides3(delta)
    else:
        p.dt_w, p.dt_x = _lib.ptr(dt_w), _lib.ptr(dt_x)
        p.dt_w_ld, p.dt_x_sb, p.dt_x_sl, p.dt_rank = dt_w.stride(0), dt_x.stride(0), dt_x.stride(1), dt_w.shape[1]
    if z_btk is not None:
        p.z = _lib.ptr(z_btk)
        p.z_sb, p.z_sl, p.z_sbi, p.z_sd = z_btk.stride(0), z_btk.stride(1), z_btk.stride(2), 1
        p.z_batch_inner = z_btk.shape[2]
    if z is not None:
        p.z_sb, p.z_sd, p.z_sl = _strides3(z)
    p.out_sb, p.out_sd, p.out_sl = _strides3(out)
    if var_b:
        p.B_sb, p.B_sg, p.B_sn, p.B_sl = B.stride()
    if var_c:
        p.C_sb, p.C_sg, p.C_sn, p.C_sl = C.stride()
    if seqlen == 1:   # a length-1 axis satisfies both layouts; make the stride say so
        p.u_sl = p.delta_sl = p.z_sl = p.out_sl = p.B_sl = p.C_sl = 1
    p.batch, p.dim, p.seqlen, p.dstate, p.ngroups = batch, dim, seqlen, dstate, ngroups
    p.dtype, p.flags, p.ckpt_every = _lib.dt(u), flags, CKPT_EVERY
    _lib.call("zg_selective_scan_fwd", p)
    return out, last, ckpt, (u, delta, z, B, C, D, delta_bias, A)


def _scan_bwd(saved, ckpt, dout, delta_softplus, dz_out=None, z_rowmap=None):
    """Raw backward (selective_scan_cuda.bwd, selective_scan.cpp:338-492).  Returns
    du, ddelta, dA, dB, dC, dD, ddelta_bias, dz."""
    u, delta, z, B, C, D, delta_bias, A = saved
    batch, dim, seqlen = u.shape
    dstate = A.shape[1]
    var_b, var_c = B.dim() >= 3, C.dim() >= 3       # constant B / C: fp32 (dim, dstate) weights (selective_scan.cpp:238-278)
    ngroups = B.shape[1] if var_b else (C.shape[1] if var_c else 1)
    if not (var_b and var_c) and ngroups != 1:
        raise RuntimeError("selective_scan backward: a constant B or C comes with one group")

    def dense(t):      # the dstate == 16 kernel takes any strides; keep channel-first or token-major as given
        return t is None or t.stride(2) == 1 or t.stride(1) == 1
    # (it also needs A and the checkpoints 16-byte aligned, scan_bwd_q4_fits; a contiguous A view 4 bytes off goes generic)
    if (dstate == 16 and var_b and var_c and A.data_ptr() % 16 == 0 and ckpt.data_ptr() % 16 == 0
            and all(dense(t) for t in (u, delta, z, dout))):
        fmt = torch.preserve_format
    else:              # generic kernel: a thread walks its own row, rows must be seq-contiguous
        def seqc(t):
            return t if (t is None or t.stride(2) == 1) else t.contiguous()
        u, delta, z, dout = seqc(u), seqc(delta), seqc(z), seqc(dout)
        B = (B if B.stride(3) == 1 else B.contiguous()) if var_b else B.contiguous()
        C = (C if C.stride(3) == 1 else C.contiguous()) if var_c else C.contiguous()
        fmt = torch.contiguous_format
    dev = u.device
    du, ddelta = torch.empty_like(u, memory_format=fmt), torch.empty_like(delta, memory_format=fmt)
    dz = None
    if z is not None:
        dz = dz_out if dz_out is not None else torch.empty_like(z, memory_format=fmt)
    dA = torch.zeros((dim, dstate), dtype=torch.float32, device=dev)
    dD = torch.zeros((dim,), dtype=torch.float32, device=dev)
    dbias = torch.zeros((dim,), dtype=torch.float32, device=dev)
    dB = torch.zeros((batch, ngroups, dstate, seqlen) if var_b else (dim, dstate), dtype=torch.float32, device=dev)
    dC = torch.zeros((batch, ngroups, dstate, seqlen) if var_c else (dim, dstate), dtype=torch.float32, device=dev)

    q = _lib.ScanBwdParams()
    p = q.fwd
    p.u, p.delta, p.z, p.B, p.C = _lib.ptr(u), _lib.ptr(delta), _lib.ptr(z), _lib.ptr(B), _lib.ptr(C)
    p.A, p.D, p.delta_bias = _lib.ptr(A), _lib.ptr(D), _lib.ptr(delta_bias)
    p.ckpt = _lib.ptr(ckpt)
    p.z_rowmap = _lib.ptr(z_rowmap)     # z read / dz written in token order (dstate == 16 kernel only)
    p.u_sb, p.u_sd, p.u_sl = _strides3(u)
    p.delta_sb, p.delta_sd, p.delta_sl = _strides3(delta)
    if z is not None:
        p.z_sb, p.z_sd, p.z_sl = _strides3(z)
    if var_b:
        p.B_sb, p.B_sg, p.B_sn, p.B_sl = B.stride()
    if var_c:
        p.C_sb, p.C_sg, p.C_sn, p.C_sl = C.stride()
    p.batch, p.dim, p.seqlen, p.dstate, p.ngroups = batch, dim, seqlen, dstate, ngroups
    p.dtype, p.ckpt_every = _lib.dt(u), CKPT_EVERY
    p.flags = (_lib.SCAN_DELTA_SOFTPLUS if delta_softplus else 0) | (_lib.SCAN_VARIABLE_B if var_b else 0) | (_lib.SCAN_VARIABLE_C if var_c else 0)
    q.dout = _lib.ptr(dout)
    q.dout_sb, q.dout_sd, q.dout_sl = _strides3(dout)
    q.du, q.ddelta, q.dz = _lib.ptr(du), _lib.ptr(ddelta), _lib.ptr(dz)
    q.du_sb, q.du_sd, q.du_sl = _strides3(du)
    q.ddelta_sb, q.ddelta_sd, q.ddelta_sl = _strides3(ddelta)
    if dz is not None:
        q.dz_sb, q.dz_sd, q.dz_sl = _strides3(dz)
    q.dA, q.dD, q.ddelta_bias, q.dB, q.dC = _lib.ptr(dA), _lib.ptr(dD), _lib.ptr(dbias), _lib.ptr(dB), _lib.ptr(dC)
    _lib.call_bwd("zg_selective_scan_bwd", q)
    return du, ddelta, dA, dB, dC, dD, dbias, dz


class SelectiveScanFn(torch.autograd.Function):
    """selective_scan_interface.py:14-74."""

    @staticmethod
    def forward(ctx, u, delta, A, B, C, D=None, z=None, delta_bias=None, delta_softplus=False,
                return_last_state=False):
        ctx.squeeze_B = B.dim() == 3
        ctx.squeeze_C = C.dim() == 3
        if ctx.squeeze_B:
            B = B.unsqueeze(1)
        if ctx.squeeze_C:
            C = C.unsqueeze(1)
        need_grad = any(t is not None and t.requires_grad for t in (u, delta, A, B, C, D, z, delta_bias))
        out, last, ckpt, saved = _scan_fwd(u, delta, A, B, C, D, z, delta_bias, delta_softplus,
                                           want_last_state=True, want_ckpt=need_grad)
        ctx.delta_softplus = delta_softplus
        ctx.has_D, ctx.has_z, ctx.has_bias = D is not None, z is not None, delta_bias is not None
        if need_grad:
            # (autograd's own storage: version checks catch an in-place change between forward and backward, saved-tensor hooks
            # and checkpointing see the tensors)
            ctx.save_for_backward(*saved, ckpt)
        if return_last_state:
            ctx.mark_non_differentiable(last)
            return out, last
        return out

    @staticmethod
    def backward(ctx, dout, *args):
        *saved, ckpt = ctx.saved_tensors
        du, ddelta, dA, dB, dC, dD, dbias, dz = _scan_bwd(tuple(saved), ckpt, dout, ctx.delta_softplus)
        dB = dB.to(saved[3].dtype)          # the activation dtype for input-dependent B / C, fp32 for constant ones
        dC = dC.to(saved[4].dtype)
        if ctx.squeeze_B:
            dB = dB.squeeze(1)
        if ctx.squeeze_C:
            dC = dC.squeeze(1)
        return (du, ddelta, dA, dB, dC, dD if ctx.has_D else None, dz if ctx.has_z else None,
                dbias if ctx.has_bias else None, None, None)


def selective_scan_fn(u, delta, A, B, C, D=None, z=None, delta_bias=None, delta_softplus=False,
                      return_last_state=False):
    """if return_last_state is True, returns (out, last_state); last_state is (batch, dim, dstate)
    fp32 and carries no gradient (selective_scan_interface.py:77-83)."""
    return SelectiveScanFn.apply(u, delta, A, B, C, D, z, delta_bias, delta_softplus, return_last_state)


# ------------------------------------------------------------------------------------------------
def _inner_fwd(xz, conv1d_weight, conv1d_bias, x_proj_weight, delta_proj_weight, A, B, C, D,
               delta_bias, B_proj_bias, C_proj_bias, delta_softplus, need_grad):
    """Shared forward of MambaInnerFn / MambaInnerFnNoOutProj (selective_scan_interface.py:296-356)
    in the reference's channel-first layout."""
    L = xz.shape[-1]
    R = delta_proj_weight.shape[1]
    N = A.shape[-1]
    if torch.is_autocast_enabled():
        x_proj_weight = x_proj_weight.to(dtype=torch.get_autocast_dtype('cuda'))
        delta_proj_weight = delta_proj_weight.to(dtype=torch.get_autocast_dtype('cuda'))
    if xz.stride(-1) != 1:
        xz = xz.contiguous()
    conv_w = conv1d_weight.reshape(conv1d_weight.shape[0], conv1d_weight.shape[-1])
    x, z = xz.chunk(2, dim=1)
    conv1d_bias = conv1d_bias.contiguous() if conv1d_bias is not None else None
    conv_out = _conv_fwd(x, conv_w, conv1d_bias, True)
    bt = xz.shape[0]
    x_dbl = F.linear(conv_out.transpose(1, 2).reshape(bt * L, -1), x_proj_weight)       # (b l) (R + 2N)
    delta = (delta_proj_weight @ x_dbl[:, :R].t()).reshape(-1, bt, L).transpose(0, 1)  # view (b, d, l)
    var_b, var_c = B is None, C is None
    if var_b:
        B = x_dbl[:, R:R + N]
        if B_proj_bias is not None:
            B = B + B_proj_bias.to(dtype=B.dtype)
        B = B.reshape(bt, L, N).permute(0, 2, 1).unsqueeze(1).contiguous()           # (b, 1, N, l)
    elif B.stride(-1) != 1:
        B = B.contiguous()
    if var_c:
        C = x_dbl[:, -N:]
        if C_proj_bias is not None:
            C = C + C_proj_bias.to(dtype=C.dtype)
        C = C.reshape(bt, L, N).permute(0, 2, 1).unsqueeze(1).contiguous()
    elif C.stride(-1) != 1:
        C = C.contiguous()
    if D is not None:
        D = D.contiguous()
    out_z, _, ckpt, saved = _scan_fwd(conv_out, delta, A, B, C, D, z, delta_bias, delta_softplus,
                                      want_last_state=False, want_ckpt=need_grad)
    return xz, conv_w, conv1d_bias, x_dbl, x_proj_weight, delta_proj_weight, conv_out, delta, B, C, D, out_z, ckpt, var_b, var_c


def _inner_bwd(ctx, dout_y, out_proj_weight=None, dout_flat=None):
    """Backward shared by the two inner functions (selective_scan_interface.py:367-434).
    dout_y: gradient wrt the scan output (b, d, l)."""
    (xz, conv_w, conv_b, x_dbl, x_proj_weight, delta_proj_weight, A, B, C, D, delta_bias, ckpt) = ctx.saved_tensors[:12]
    bt, _, L = xz.shape
    R = delta_proj_weight.shape[1]
    N = A.shape[-1]
    x, z = xz.chunk(2, dim=1)
    # checkpoint_lvl = 1: recompute conv output and delta (selective_scan_interface.py:379-382)
    conv_out = _conv_fwd(x, conv_w, conv_b, True)
    delta = (delta_proj_weight @ x_dbl[:, :R].t()).reshape(-1, bt, L).transpose(0, 1)
    dxz = torch.empty_like(xz)
    dx, dz = dxz.chunk(2, dim=1)
    dconv_out, ddelta, dA, dB, dC, dD, ddelta_bias, dz_ = _scan_bwd(
        (conv_out, delta, z, B, C, D, delta_bias, A), ckpt, dout_y, ctx.delta_softplus, dz_out=dz)
    dx_dbl = torch.empty_like(x_dbl)
    dB_proj_bias = dC_proj_bias = None
    dB_ret = dC_ret = None
    if ctx.var_b:
        dBm = dB.squeeze(1).permute(0, 2, 1).reshape(bt * L, N)
        dB_proj_bias = dBm.sum(0) if ctx.has_B_bias else None
        dx_dbl[:, R:R + N] = dBm
    else:
        dB_ret = dB
    if ctx.var_c:
        dCm = dC.squeeze(1).permute(0, 2, 1).reshape(bt * L, N)
        dC_proj_bias = dCm.sum(0) if ctx.has_C_bias else None
        dx_dbl[:, -N:] = dCm
    else:
        dC_ret = dC
    ddelta2 = ddelta.transpose(0, 1).reshape(ddelta.shape[1], bt * L)                     # d (b l)
    ddelta_proj_weight = ddelta2.to(x_dbl.dtype) @ x_dbl[:, :R]
    dx_dbl[:, :R] = ddelta2.t().to(delta_proj_weight.dtype) @ delta_proj_weight
    conv_flat = conv_out.transpose(1, 2).reshape(bt * L, -1)
    dx_proj_weight = dx_dbl.t() @ conv_flat
    dconv_flat = dconv_out.transpose(1, 2).reshape(bt * L, -1) + dx_dbl @ x_proj_weight
    dconv = dconv_flat.reshape(bt, L, -1).transpose(1, 2)
    dx_, dconv_w, dconv_b = _conv_bwd(x, conv_w, conv_b, dconv, True, dx_out=dx)
    return (dxz, dconv_w.reshape(conv_w.shape[0], 1, -1).to(conv_w.dtype), dconv_b.to(conv_b.dtype) if conv_b is not None else None,
            dx_proj_weight, ddelta_proj_weight, dA, dB_ret, dC_ret,
            dD if D is not None else None, ddelta_bias if delta_bias is not None else None,
            dB_proj_bias, dC_proj_bias)


class MambaInnerFnNoOutProj(torch.autograd.Function):
    """selective_scan_interface.py:155-289.  Returns out_z (batch, dim, seqlen)."""

    @staticmethod
    def forward(ctx, xz, conv1d_weight, conv1d_bias, x_proj_weight, delta_proj_weight,
                A, B=None, C=None, D=None, delta_bias=None, B_proj_bias=None, C_proj_bias=None,
                delta_softplus=True, checkpoint_lvl=1):
        assert checkpoint_lvl in [0, 1]
        need_grad = any(t is not None and t.requires_grad for t in
                        (xz, conv1d_weight, conv1d_bias, x_proj_weight, delta_proj_weight, A, B, C, D, delta_bias))
        (xz, conv_w, conv_b, x_dbl, xw, dw, conv_out, delta, Bm, Cm, D, out_z, ckpt, var_b, var_c) = _inner_fwd(
            xz, conv1d_weight, conv1d_bias, x_proj_weight, delta_proj_weight, A, B, C, D, delta_bias,
            B_proj_bias, C_proj_bias, delta_softplus, need_grad)
        ctx.delta_softplus = delta_softplus
        ctx.var_b, ctx.var_c = var_b, var_c
        ctx.has_B_bias, ctx.has_C_bias = B_proj_bias is not None, C_proj_bias is not None
        if need_grad:
            ctx.save_for_backward(xz, conv_w, conv_b, x_dbl, xw, dw, A, Bm, Cm, D, delta_bias, ckpt)
        return out_z

    @staticmethod
    def backward(ctx, dout):
        g = _inner_bwd(ctx, dout)
        (dxz, dcw, dcb, dxw, ddw, dA, dB, dC, dD, dbias, dBb, dCb) = g
        return (dxz, dcw, dcb, dxw, ddw, dA, dB, dC, dD, dbias, dBb, dCb, None, None)


class MambaInnerFn(torch.autograd.Function):
    """selective_scan_interface.py:292-434.  Returns (batch, seqlen, d_model)."""

    @staticmethod
    def forward(ctx, xz, conv1d_weight, conv1d_bias, x_proj_weight, delta_proj_weight,
                out_proj_weight, out_proj_bias, A, B=None, C=None, D=None, delta_bias=None,
                B_proj_bias=None, C_proj_bias=None, delta_softplus=True, checkpoint_lvl=1):
        assert checkpoint_lvl in [0, 1]
        if torch.is_autocast_enabled():
            out_proj_weight = out_proj_weight.to(dtype=torch.get_autocast_dtype('cuda'))
            out_proj_bias = out_proj_bias.to(dtype=torch.get_autocast_dtype('cuda')) if out_proj_bias is not None else None
        need_grad = any(t is not None and t.requires_grad for t in
                        (xz, conv1d_weight, conv1d_bias, x_proj_weight, delta_proj_weight, out_proj_weight,
                         out_proj_bias, A, B, C, D, delta_bias))
        (xz, conv_w, conv_b, x_dbl, xw, dw, conv_out, delta, Bm, Cm, D, out_z, ckpt, var_b, var_c) = _inner_fwd(
            xz, conv1d_weight, conv1d_bias, x_proj_weight, delta_proj_weight, A, B, C, D, delta_bias,
            B_proj_bias, C_proj_bias, delta_softplus, need_grad)
        ctx.delta_softplus = delta_softplus
        ctx.var_b, ctx.var_c = var_b, var_c
        ctx.has_B_bias, ctx.has_C_bias = B_proj_bias is not None, C_proj_bias is not None
        ctx.has_out_bias = out_proj_bias is not None
        if need_grad:
            # (out_z: the reference recomputes it in the bwd kernel; keeping it costs B*E*L*2 bytes)
            ctx.save_for_backward(xz, conv_w, conv_b, x_dbl, xw, dw, A, Bm, Cm, D, delta_bias, ckpt, out_proj_weight, out_z)
        return F.linear(out_z.transpose(1, 2), out_proj_weight, out_proj_bias)

    @staticmethod
    def backward(ctx, dout):
        W, out_z = ctx.saved_tensors[12:14]
        bt, L, Dm = dout.shape
        dout2 = dout.reshape(bt * L, Dm)
        dout_y = (dout2 @ W).reshape(bt, L, -1).transpose(1, 2)                      # (b, d, l)
        dW = dout2.t() @ out_z.transpose(1, 2).reshape(bt * L, -1)
        dbias = dout2.sum(0) if ctx.has_out_bias else None
        (dxz, dcw, dcb, dxw, ddw, dA, dB, dC, dD, dbias_dt, dBb, dCb) = _inner_bwd(ctx, dout_y)
        return (dxz, dcw, dcb, dxw, ddw, dW, dbias, dA, dB, dC, dD, dbias_dt, dBb, dCb, None, None)


# ------------------------------------------------------------------------------------------------
# Token-major training core: what MambaInnerFn computes between in_proj and out_proj, but laid out the
# way the sampling engine runs it -- activations (batch * seqlen, channels) row-major, the zigzag
# permutation never materialised (the conv gathers x rows, the scan gathers z rows through the path
# table; the backward scatters dx / dz rows back through the same table).  No transposed copies, no
# index_select in either direction.
def _tok_linear(x, w):
    """x (M, K) @ w(N, K)^T on the wgmma kernel for bf16, cuBLAS otherwise."""
    if x.dtype == torch.bfloat16 and w.dtype == torch.bfloat16 and x.is_cuda:
        from .engine import _linear
        return _linear(x, w)
    return F.linear(x, w)


def _tok_core_fwd(xz, conv_w, conv_b, x_proj_w, dt_proj_w, A, D, delta_bias, rowmap, bt, L, want_ckpt):
    from .causal_conv1d_interface import _conv_fwd
    E = xz.shape[1] // 2
    R, N = dt_proj_w.shape[1], A.shape[1]
    xz3 = xz.view(bt, L, 2 * E)
    x_log = xz3[:, :, :E].transpose(1, 2)             # logical (bt, E, L), channel stride 1
    z_log = xz3[:, :, E:].transpose(1, 2)
    xc = _conv_fwd(x_log, conv_w, conv_b, True, x_rowmap=rowmap)                # token-major memory, scan order
    xc_flat = xc.transpose(1, 2).reshape(bt * L, E)
    x_dbl = _tok_linear(xc_flat, x_proj_w)                                       # (bt L, R + 2N)
    delta = _tok_linear(x_dbl[:, :R], dt_proj_w)                                 # (bt L, E)
    d_log = delta.view(bt, L, E).transpose(1, 2)
    xd3 = x_dbl.view(bt, L, R + 2 * N)
    B_log = xd3[:, :, R:R + N].permute(0, 2, 1).unsqueeze(1)                     # (bt, 1, N, L) views
    C_log = xd3[:, :, R + N:].permute(0, 2, 1).unsqueeze(1)
    y, _, ckpt, _ = _scan_fwd(xc, d_log, A, B_log, C_log, D, z_log, delta_bias, True, z_rowmap=rowmap,
                              want_last_state=False, want_ckpt=want_ckpt)
    return y, ckpt, x_dbl, (x_log, z_log, xc, xc_flat, d_log, B_log, C_log)


class MambaInnerTokFn(torch.autograd.Function):
    """xz (batch * seqlen, 2 * d_inner) token-major, TOKEN order -> y (batch * seqlen, d_inner) in SCAN
    order (scan position l holds token rowmap[l]; rowmap None = identity).  Same math as
    MambaInnerFnNoOutProj (selective_scan_interface.py:155-289 of the reference) applied to
    xz[:, :, rowmap]; checkpoint_lvl-1 style: the conv output and delta are recomputed in the backward."""

    @staticmethod
    def forward(ctx, xz, conv1d_weight, conv1d_bias, x_proj_weight, delta_proj_weight, A, D, delta_bias, rowmap, bt, L):
        if torch.is_autocast_enabled():
            x_proj_weight = x_proj_weight.to(dtype=torch.get_autocast_dtype('cuda'))
            delta_proj_weight = delta_proj_weight.to(dtype=torch.get_autocast_dtype('cuda'))
        if not xz.is_contiguous():
            xz = xz.contiguous()
        conv_w = conv1d_weight.reshape(conv1d_weight.shape[0], conv1d_weight.shape[-1]).contiguous()
        conv_b = conv1d_bias.contiguous() if conv1d_bias is not None else None
        need_grad = any(t is not None and t.requires_grad for t in
                        (xz, conv1d_weight, conv1d_bias, x_proj_weight, delta_proj_weight, A, D, delta_bias))
        y, ckpt, x_dbl, _ = _tok_core_fwd(xz, conv_w, conv_b, x_proj_weight, delta_proj_weight, A, D, delta_bias,
                                          rowmap, bt, L, need_grad)
        if need_grad:
            ctx.save_for_backward(xz, conv_w, conv_b, x_dbl, x_proj_weight, delta_proj_weight, A, D, delta_bias, ckpt, rowmap)
            ctx.dims = (bt, L)
            ctx.wshape = conv1d_weight.shape
        return y.transpose(1, 2).reshape(bt * L, -1)

    @staticmethod
    def backward(ctx, dy):
        from .causal_conv1d_interface import _conv_fwd, _conv_bwd
        (xz, conv_w, conv_b, x_dbl, x_proj_w, dt_proj_w, A, D, delta_bias, ckpt, rowmap) = ctx.saved_tensors
        bt, L = ctx.dims
        E = xz.shape[1] // 2
        R, N = dt_proj_w.shape[1], A.shape[1]
        xz3 = xz.view(bt, L, 2 * E)
        x_log, z_log = xz3[:, :, :E].transpose(1, 2), xz3[:, :, E:].transpose(1, 2)
        xc = _conv_fwd(x_log, conv_w, conv_b, True, x_rowmap=rowmap)             # recompute (cheap, saves 2 E bytes / token)
        xc_flat = xc.transpose(1, 2).reshape(bt * L, E)
        delta = _tok_linear(x_dbl[:, :R], dt_proj_w)
        d_log = delta.view(bt, L, E).transpose(1, 2)
        xd3 = x_dbl.view(bt, L, R + 2 * N)
        B_log = xd3[:, :, R:R + N].permute(0, 2, 1).unsqueeze(1)
        C_log = xd3[:, :, R + N:].permute(0, 2, 1).unsqueeze(1)
        dxz = torch.empty_like(xz)
        dxz3 = dxz.view(bt, L, 2 * E)
        dx_log, dz_log = dxz3[:, :, :E].transpose(1, 2), dxz3[:, :, E:].transpose(1, 2)
        dy_log = dy.contiguous().view(bt, L, E).transpose(1, 2)
        du, ddelta, dA, dB, dC, dD, dbias, _ = _scan_bwd((xc, d_log, z_log, B_log, C_log, D, delta_bias, A), ckpt, dy_log,
                                                         True, dz_out=dz_log, z_rowmap=rowmap)
        ddelta_flat = ddelta.transpose(1, 2).reshape(bt * L, E)
        dx_dbl = torch.empty_like(x_dbl)
        dx_dbl[:, :R] = ddelta_flat @ dt_proj_w
        dx_dbl[:, R:R + N] = dB.squeeze(1).transpose(1, 2).reshape(bt * L, N)
        dx_dbl[:, R + N:] = dC.squeeze(1).transpose(1, 2).reshape(bt * L, N)
        d_dt_w = ddelta_flat.t() @ x_dbl[:, :R]
        d_x_w = dx_dbl.t() @ xc_flat
        dxc = torch.addmm(du.transpose(1, 2).reshape(bt * L, E), dx_dbl, x_proj_w)
        _, dcw, dcb = _conv_bwd(x_log, conv_w, conv_b, dxc.view(bt, L, E).transpose(1, 2), True, dx_out=dx_log, x_rowmap=rowmap)
        return (dxz, dcw.reshape(ctx.wshape).to(conv_w.dtype), dcb.to(conv_b.dtype) if conv_b is not None else None,
                d_x_w, d_dt_w, dA, dD if D is not None else None, dbias if delta_bias is not None else None, None, None, None)


def mamba_inner_tok_fn(xz, conv1d_weight, conv1d_bias, x_proj_weight, delta_proj_weight, A, D, delta_bias, rowmap, bt, L):
    return MambaInnerTokFn.apply(xz, conv1d_weight, conv1d_bias, x_proj_weight, delta_proj_weight, A, D, delta_bias, rowmap, bt, L)


def mamba_inner_fn(xz, conv1d_weight, conv1d_bias, x_proj_weight, delta_proj_weight,
                   out_proj_weight, out_proj_bias, A, B=None, C=None, D=None, delta_bias=None,
                   B_proj_bias=None, C_proj_bias=None, delta_softplus=True):
    return MambaInnerFn.apply(xz, conv1d_weight, conv1d_bias, x_proj_weight, delta_proj_weight,
                              out_proj_weight, out_proj_bias, A, B, C, D, delta_bias,
                              B_proj_bias, C_proj_bias, delta_softplus)


def mamba_inner_fn_no_out_proj(xz, conv1d_weight, conv1d_bias, x_proj_weight, delta_proj_weight,
                               A, B=None, C=None, D=None, delta_bias=None, B_proj_bias=None,
                               C_proj_bias=None, delta_softplus=True):
    return MambaInnerFnNoOutProj.apply(xz, conv1d_weight, conv1d_bias, x_proj_weight, delta_proj_weight,
                                       A, B, C, D, delta_bias, B_proj_bias, C_proj_bias, delta_softplus)


def bimamba_inner_fn(xz, conv1d_weight, conv1d_bias, x_proj_weight, delta_proj_weight,
                     out_proj_weight, out_proj_bias, A, A_b, B=None, C=None, D=None, delta_bias=None,
                     B_proj_bias=None, C_proj_bias=None, delta_softplus=True):
    """selective_scan_interface.py:437-603 (unused by ZigMa; composed from the ops above): shared
    conv / projections, forward scan with A plus a scan of the flipped sequence with A_b, summed
    before out_proj."""
    L = xz.shape[-1]
    R = delta_proj_weight.shape[1]
    N = A.shape[-1]
    from .causal_conv1d_interface import causal_conv1d_fn
    x, z = xz.chunk(2, dim=1)
    bt = xz.shape[0]
    xc = causal_conv1d_fn(x, conv1d_weight.reshape(conv1d_weight.shape[0], -1), conv1d_bias, "silu")
    x_dbl = F.linear(xc.transpose(1, 2).reshape(bt * L, -1), x_proj_weight)
    delta = (delta_proj_weight @ x_dbl[:, :R].t()).reshape(-1, bt, L).transpose(0, 1)
    if B is None:
        B = x_dbl[:, R:R + N]
        if B_proj_bias is not None:
            B = B + B_proj_bias.to(dtype=B.dtype)
        B = B.reshape(bt, L, N).permute(0, 2, 1).contiguous()
    if C is None:
        C = x_dbl[:, -N:]
        if C_proj_bias is not None:
            C = C + C_proj_bias.to(dtype=C.dtype)
        C = C.reshape(bt, L, N).permute(0, 2, 1).contiguous()
    y = selective_scan_fn(xc, delta, A, B, C, D, z=z, delta_bias=delta_bias, delta_softplus=delta_softplus)
    y_b = selective_scan_fn(xc.flip([-1]), delta.flip([-1]), A_b, B.flip([-1]), C.flip([-1]), D,
                            z.flip([-1]), delta_bias, delta_softplus=delta_softplus)
    return F.linear((y + y_b.flip([-1])).transpose(1, 2), out_proj_weight, out_proj_bias)
