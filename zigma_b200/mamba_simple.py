"""ZigMa's Mamba mixer (``dis_mamba/mamba_ssm/modules/mamba_simple.py`` of the reference) on the
sm_90a kernels.  Same constructor arguments, parameter names / shapes / init and scan-type
dispatch (:64-268, :274-444); the single-token ``step`` / inference cache (:445-608) is out of
scope (diffusion never decodes token by token).

Two execution paths share the parameters:
  * ``forward`` -- autograd-capable, channel-first like the reference (in_proj -> permutation
    gather -> ``mamba_inner_fn`` -> scatter), built on ``selective_scan_interface``;
  * ``engine.ZigMaEngine`` (sampling) reads the same parameters but runs token-major with no
    permuted copy: the conv kernel gathers x rows and the scan kernel gathers z rows through the
    path table, and the scatter back is folded into the fused block tail.
"""
import math

import torch
import torch.nn as nn
import torch.nn.functional as F

import os

from .selective_scan_interface import mamba_inner_fn, mamba_inner_fn_no_out_proj, mamba_inner_tok_fn, selective_scan_fn


_INV_CACHE = {}


def _inverse_of(perm):
    """Inverse permutation, or None when ``perm`` is not a bijection of range(len) (cached per tensor)."""
    key = (perm.data_ptr(), perm.numel(), str(perm.device))
    hit = _INV_CACHE.get(key)
    if hit is None or hit[0] is not perm:
        n = perm.numel()
        ok = bool(n) and bool(((perm >= 0) & (perm < n)).all()) and int(torch.unique(perm).numel()) == n
        inv = None
        if ok:
            inv = torch.empty_like(perm)
            inv[perm] = torch.arange(n, device=perm.device, dtype=perm.dtype)
        if len(_INV_CACHE) > 256:
            _INV_CACHE.clear()
        hit = _INV_CACHE[key] = (perm, inv)
    return hit[1]


class _PermuteFn(torch.autograd.Function):
    """y = x.index_select(dim, perm) for a PERMUTATION perm: the backward is the gather by the inverse
    permutation.  The reference writes ``x[:, :, perm]`` (mamba_simple.py:56,61), whose autograd
    backward is a sort-based index_put with accumulation -- 8 ms per layer at the config-2 shape,
    a large share of a training step -- although no index repeats."""

    @staticmethod
    def forward(ctx, x, perm, inv, dim):
        ctx.inv, ctx.dim = inv, dim
        return x.index_select(dim, perm)

    @staticmethod
    def backward(ctx, g):
        return g.index_select(ctx.dim, ctx.inv), None, None, None


def permute_along(x, perm, dim):
    """x gathered along ``dim`` by ``perm`` (contiguous result), with the cheap permutation backward when
    perm is a bijection and plain advanced indexing otherwise."""
    inv = _inverse_of(perm) if (x.requires_grad and torch.is_grad_enabled()) else None
    if inv is not None:
        return _PermuteFn.apply(x, perm, inv, dim)
    return x.index_select(dim, perm)


def forward_permutation(xz_main, _perm):
    return permute_along(xz_main, _perm, 2)  # [B, C, T]


def backward_permutation(o_main, _perm_rev):
    return permute_along(o_main, _perm_rev, 1)  # [B, T, C]


def _is_video(scan_type):
    return scan_type.startswith("video_") or scan_type.startswith("zzvideo_")


class Mamba(nn.Module):
    def __init__(self, d_model, d_state=16, d_conv=4, expand=2, dt_rank="auto", dt_min=0.001, dt_max=0.1,
                 dt_init="random", dt_scale=1.0, dt_init_floor=1e-4, conv_bias=True, bias=False,
                 use_fast_path=True, layer_idx=None, device=None, dtype=None, scan_type="v2", **kwargs):
        fk = {"device": device, "dtype": dtype}
        super().__init__()
        self.d_model, self.d_state, self.d_conv, self.expand = d_model, d_state, d_conv, expand
        self.d_inner = int(expand * d_model)
        self.dt_rank = math.ceil(d_model / 16) if dt_rank == "auto" else dt_rank
        self.use_fast_path = use_fast_path
        self.layer_idx = layer_idx
        self.scan_type = scan_type
        # NB the reference's ZigMa hands scan_type="zzvideo_*" to a Mamba that only accepts the
        # "video_" prefix (mamba_simple.py:164-171 vs model_zigma.py:746,807), so its 3-D configs
        # cannot be constructed as shipped; both spellings are accepted here.
        if not (scan_type in ("v1", "v2") or _is_video(scan_type)
                or any(scan_type.startswith(p) for p in ("zigzagN", "hilbertN", "randomN", "parallelN"))):
            raise AssertionError(f"Invalid scan_type: {scan_type}")
        if scan_type.startswith("parallelN"):
            raise NotImplementedError("parallelN has no forward branch in the reference either (mamba_simple.py:443-444)")

        self.in_proj = nn.Linear(d_model, self.d_inner * 2, bias=bias, **fk)
        self.conv1d = nn.Conv1d(self.d_inner, self.d_inner, kernel_size=d_conv, groups=self.d_inner,
                                padding=d_conv - 1, bias=conv_bias, **fk)
        self.zigzag_paths = kwargs.get("zigzag_paths", None)
        self.zigzag_paths_reverse = kwargs.get("zigzag_paths_reverse", None)
        self.video_frames = kwargs.get("video_frames", None)
        self.st_order = kwargs.get("st_order", None)
        self.extras = kwargs.get("extras", None)
        self.use_jit = kwargs.get("use_jit", False)
        self.activation = "silu"
        self.act = nn.SiLU()
        self.x_proj = nn.Linear(self.d_inner, self.dt_rank + d_state * 2, bias=False, **fk)
        self.dt_proj = nn.Linear(self.dt_rank, self.d_inner, bias=True, **fk)

        # dt projection init preserving variance; bias = softplus^-1(dt), dt log-uniform in
        # [dt_min, dt_max] (mamba_simple.py:128-148)
        std = self.dt_rank ** -0.5 * dt_scale
        if dt_init == "constant":
            nn.init.constant_(self.dt_proj.weight, std)
        elif dt_init == "random":
            nn.init.uniform_(self.dt_proj.weight, -std, std)
        else:
            raise NotImplementedError
        dt = torch.exp(torch.rand(self.d_inner, **fk) * (math.log(dt_max) - math.log(dt_min))
                       + math.log(dt_min)).clamp(min=dt_init_floor)
        with torch.no_grad():
            self.dt_proj.bias.copy_(dt + torch.log(-torch.expm1(-dt)))
        self.dt_proj.bias._no_reinit = True

        def s4d_real_log():
            return torch.log(torch.arange(1, d_state + 1, dtype=torch.float32, device=device)
                             .repeat(self.d_inner, 1).contiguous())
        self.A_log = nn.Parameter(s4d_real_log())
        self.A_log._no_weight_decay = True
        self.D = nn.Parameter(torch.ones(self.d_inner, device=device))
        self.D._no_weight_decay = True

        if scan_type == "v2":   # second parameter set for the backward sweep (:229-264)
            self.A_b_log = nn.Parameter(s4d_real_log())
            self.A_b_log._no_weight_decay = True
            self.conv1d_b = nn.Conv1d(self.d_inner, self.d_inner, kernel_size=d_conv, groups=self.d_inner,
                                      padding=d_conv - 1, bias=conv_bias, **fk)
            self.x_proj_b = nn.Linear(self.d_inner, self.dt_rank + d_state * 2, bias=False, **fk)
            self.dt_proj_b = nn.Linear(self.dt_rank, self.d_inner, bias=True, **fk)
            self.D_b = nn.Parameter(torch.ones(self.d_inner, device=device))
            self.D_b._no_weight_decay = True

        self.out_proj = nn.Linear(self.d_inner, d_model, bias=bias, **fk)

    # --------------------------------------------------------------------------------------------
    def forward(self, hidden_states, inference_params=None):
        if inference_params is not None:
            raise NotImplementedError("zigma_b200: the autoregressive inference cache / step() is out of scope")
        return self._mamba_inner_forward(hidden_states)

    def _inner_args(self, suffix=""):
        """Parameter set of the forward sweep ("") or of v2's backward sweep ("_b")."""
        conv, xp, dp = getattr(self, "conv1d" + suffix), getattr(self, "x_proj" + suffix), getattr(self, "dt_proj" + suffix)
        A_log = self.A_b_log if suffix else self.A_log
        D = self.D_b if suffix else self.D
        return dict(conv1d_weight=conv.weight, conv1d_bias=conv.bias, x_proj_weight=xp.weight,
                    delta_proj_weight=dp.weight, A=-torch.exp(A_log.float()), D=D.float(),
                    delta_bias=dp.bias.float())

    # ---- token-major path (training and eager inference): no transposes, permutation fused into the kernels ----
    def _tok_eligible(self, hidden_states):
        st = self.scan_type
        return (self.use_fast_path and hidden_states.is_cuda and self.d_state == 16 and not (self.extras or 0)
                and (st == "v1" or (not _is_video(st) and st != "v2"))
                and os.environ.get("ZIGMA_TOKEN_MAJOR_TRAIN", "1") != "0")

    def _rowmap32(self, perm):
        cache = self.__dict__.setdefault("_rowmap_cache", {})
        key = (perm.data_ptr(), str(perm.device))
        hit = cache.get(key)
        if hit is None or hit[0] is not perm:
            hit = cache[key] = (perm, perm.to(torch.int32).contiguous())
        return hit[1]

    def _tok_forward(self, hidden_states, scan_order=False):
        """Same function as the channel-first branch below for v1 / zigzagN / hilbertN / randomN:
        in_proj -> [gather by perm] -> conv -> x_proj / dt_proj -> scan * silu(z) -> out_proj -> [gather by
        perm_rev], with the two gathers folded into the conv / scan kernels (forward and backward)."""
        batch, seqlen, dm = hidden_states.shape
        a = self._inner_args()
        xz = F.linear(hidden_states.reshape(batch * seqlen, dm), self.in_proj.weight, self.in_proj.bias)
        perm = perm_rev = None
        if self.scan_type != "v1":
            perm = self.zigzag_paths[self.layer_idx]
            perm_rev = self.zigzag_paths_reverse[self.layer_idx]
            if perm.device != xz.device:
                perm, perm_rev = perm.to(xz.device), perm_rev.to(xz.device)
        y = mamba_inner_tok_fn(xz, a["conv1d_weight"], a["conv1d_bias"], a["x_proj_weight"], a["delta_proj_weight"],
                               a["A"], a["D"], a["delta_bias"], None if perm is None else self._rowmap32(perm), batch, seqlen)
        out = F.linear(y, self.out_proj.weight, self.out_proj.bias).view(batch, seqlen, -1)
        if scan_order:      # the caller folds the un-permutation into its own kernel (block tail)
            return out, (None if perm_rev is None else self._rowmap32(perm_rev))
        return out if perm_rev is None else permute_along(out, perm_rev, 1)

    def forward_scan_order(self, hidden_states):
        """(mix, rowmap): ``forward(hidden_states) == mix[:, rowmap]`` (rowmap None = identity).  For the token-major
        mixers the out_proj result is returned in SCAN order together with the int32 inverse table, so that the gather
        can be fused downstream; every other scan type returns the finished output."""
        if self._tok_eligible(hidden_states):
            return self._tok_forward(hidden_states, scan_order=True)
        return self.forward(hidden_states), None

    def _mamba_inner_forward(self, hidden_states):
        """hidden_states (B, L, D) -> (B, L, D).  mamba_simple.py:274-444."""
        batch, seqlen, _ = hidden_states.shape
        if self._tok_eligible(hidden_states):
            return self._tok_forward(hidden_states)
        # matmul and BLD -> B(2E)L transpose in one go (:290-296)
        xz = (self.in_proj.weight @ hidden_states.reshape(batch * seqlen, -1).t()).reshape(-1, batch, seqlen).transpose(0, 1)
        if self.in_proj.bias is not None:
            xz = xz + self.in_proj.bias.to(dtype=xz.dtype).view(1, -1, 1)
        if not self.use_fast_path:
            return self._slow_forward(xz, seqlen)
        a = self._inner_args()
        st = self.scan_type

        def inner(xz_):
            return mamba_inner_fn(xz_, a["conv1d_weight"], a["conv1d_bias"], a["x_proj_weight"], a["delta_proj_weight"],
                                  self.out_proj.weight, self.out_proj.bias, a["A"], None, None, a["D"],
                                  delta_bias=a["delta_bias"], delta_softplus=True)
        if st == "v1":
            return inner(xz)
        if st == "v2":
            ab = self._inner_args("_b")
            out = mamba_inner_fn_no_out_proj(xz, a["conv1d_weight"], a["conv1d_bias"], a["x_proj_weight"],
                                             a["delta_proj_weight"], a["A"], None, None, a["D"],
                                             delta_bias=a["delta_bias"], delta_softplus=True)
            out_b = mamba_inner_fn_no_out_proj(xz.flip([-1]), ab["conv1d_weight"], ab["conv1d_bias"], ab["x_proj_weight"],
                                               ab["delta_proj_weight"], ab["A"], None, None, ab["D"],
                                               delta_bias=ab["delta_bias"], delta_softplus=True)
            return F.linear((out + out_b.flip([-1])).transpose(1, 2), self.out_proj.weight, self.out_proj.bias)
        perm = self.zigzag_paths[self.layer_idx]
        perm_rev = self.zigzag_paths_reverse[self.layer_idx]
        ex = self.extras or 0
        if not _is_video(st):   # zigzagN / hilbertN / randomN (:356-395)
            xz = torch.cat([xz[:, :, :ex], forward_permutation(xz[:, :, ex:], perm)], dim=2)
            out = inner(xz)
            return torch.cat([out[:, :ex, :], backward_permutation(out[:, ex:, :], perm_rev)], dim=1)
        # video: factorised spatial / temporal scans (:396-442)
        assert ex == 0, "video_ only supports extra=0"
        T = self.video_frames
        K = seqlen // T
        s_or_t = self.st_order[self.layer_idx]
        x4 = xz.reshape(batch, -1, T, K)
        if s_or_t == "s":
            xr = x4.permute(0, 2, 1, 3).reshape(batch * T, -1, K)
        elif s_or_t == "t":
            xr = x4.permute(0, 3, 1, 2).reshape(batch * K, -1, T)
        else:
            raise NotImplementedError
        out = permute_along(inner(permute_along(xr, perm, 2)), perm_rev, 1)
        if s_or_t == "s":
            return out.reshape(batch, seqlen, -1)
        return out.reshape(batch, K, T, -1).permute(0, 2, 1, 3).reshape(batch, seqlen, -1)

    def _slow_forward(self, xz, seqlen):
        """use_fast_path=False branch (:445-490): separate conv / projections / selective_scan_fn."""
        from .causal_conv1d_interface import causal_conv1d_fn
        x, z = xz.chunk(2, dim=1)
        x = causal_conv1d_fn(x, self.conv1d.weight.reshape(self.d_inner, -1), self.conv1d.bias, self.activation)
        bt = x.shape[0]
        x_dbl = self.x_proj(x.transpose(1, 2).reshape(bt * seqlen, -1))
        dt, B, C = torch.split(x_dbl, [self.dt_rank, self.d_state, self.d_state], dim=-1)
        dt = (self.dt_proj.weight @ dt.t()).reshape(-1, bt, seqlen).transpose(0, 1)
        B = B.reshape(bt, seqlen, -1).transpose(1, 2).contiguous()
        C = C.reshape(bt, seqlen, -1).transpose(1, 2).contiguous()
        y = selective_scan_fn(x, dt, -torch.exp(self.A_log.float()), B, C, self.D.float(), z=z,
                              delta_bias=self.dt_proj.bias.float(), delta_softplus=True)
        return self.out_proj(y.transpose(1, 2))
