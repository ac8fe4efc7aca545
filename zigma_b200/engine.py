"""Inference fast path of ZigMa.forward on H100: token-major, fused, CUDA-graph capturable.

What the reference executes per block (SURVEY.md section 3.2/3.3) and what replaces it here:

  reference (channel-first, ~25 launches / block)            here (token-major, 7 launches / block)
  ---------------------------------------------------------  -----------------------------------------
  in_proj GEMM + "b l d -> d (b l)" rearranges               GEMM  modded(B*L, D) @ W_in^T -> xz(B*L, 2E)
  xz[:, :, perm].contiguous() + torch.cat  (1.3 GB / layer)  -- gone: kernels read rows through `perm`
  causal_conv1d_fwd                                          zg_causal_conv1d_fwd(x_rowmap = perm)
  x_proj GEMM, dt_proj GEMM, B/C rearrange + contiguous      2 GEMMs; B/C read in place from x_dbl rows
  selective_scan_fwd (out AND out_z written)                 zg_selective_scan_fwd(z_rowmap = perm)
  out_proj GEMM, out[:, perm_rev].contiguous() + cat         GEMM; scatter folded into the block tail
  gate*mix + x, fused add+RMSNorm (Triton), modulate         zg_block_tail_fwd (one pass)

Numerics follow the reference's bf16 path rounding for rounding (every tensor the reference
materialises in bf16 is rounded to bf16 at the same point), so results agree with the reference
to fp32-accumulation-order noise.  The dense bf16 projections run on the hand-written wgmma kernel
``zg_gemm_bf16_tn`` (``ZIGMA_TCGEN05=0`` switches them to the library GEMM for A/B timing; fp32 models always
use the library GEMM -- the tensor-core kernel is bf16 only).
"""
import os

import torch
import torch.nn.functional as F

from . import _lib
from .causal_conv1d_interface import _conv_fwd
from .selective_scan_interface import _scan_fwd


def _i32(t):
    return t.to(torch.int32).contiguous()


def _linear(x2d, weight, bias=None):
    """(M, K) @ (N, K)^T.  bf16 goes to the hand-written wgmma kernel (zg_gemm_bf16_tn; ZIGMA_TCGEN05=0, the switch's historical name, routes
    it to the library GEMM instead, e.g. for A/B timing); fp32 / fp16 always use the library GEMM."""
    if x2d.dtype == torch.bfloat16 and os.environ.get("ZIGMA_TCGEN05", "1") == "1" and x2d.stride(0) % 8 == 0 and weight.stride(0) % 8 == 0:
        from .gemm import linear_bf16
        return linear_bf16(x2d, weight, bias)
    return F.linear(x2d, weight, bias)


def fused_dt_ok(dtype, E, L, N, R, dt_w):
    """Shape class of the scan kernel's fused dt_proj prologue (include/zigma_b200.h, zg_scan_params.dt_w)."""
    return (dtype in (torch.bfloat16, torch.float16) and N == 16 and R in (40, 48) and L % 8 == 0 and E % 64 == 0
            and dt_w.dtype == dtype and dt_w.stride(1) == 1 and dt_w.stride(0) % 8 == 0 and (R + 2 * N) % 8 == 0)


def scan_hot_path_ok(dtype, E, L, N, R):
    """Shape class of zg::scan_fwd_tma_kernel as the engine calls it (B / C read in place from the x_dbl rows): the features only
    that kernel implements (OUT_REVERSE / OUT_ACCUMULATE, z_batch_inner) may be requested."""
    return (dtype in (torch.bfloat16, torch.float16) and N == 16 and L % 8 == 0 and L > 0 and E % 64 == 0 and R % 8 == 0
            and (R + 2 * N) % 8 == 0 and os.environ.get("ZG_SCAN_TMA", "1") != "0")


def block_tail(x, mix, gate, shift, scale, norm_w, residual, rowmap, eps, final=False, mod_div=1, want_modded=True, want_rstd=False,
               mix_bcast=False, path_scale=None, x_from=None):
    """zg_block_tail_fwd wrapper.  x: (Bt, L, D) contiguous; gate/shift/scale: (Bt // mod_div, D)
    views with a common row stride.  Returns residual_out (fp32), normed, modded.
    mix_bcast: ``mix`` is one (L, D) table added to every batch element (gate None = 1): the positional embedding.
    path_scale: (Bt,) drop-path multipliers in x.dtype (zg_block_tail_fwd_dp): hidden * path_scale[b] joins the residual.
    x_from = (rstd, norm_w) of the previous tail, norm_w in the activation dtype, with x None (zg_block_tail_fwd_rebuild): x is that
    tail's normed output, rebuilt from `residual` (its residual_out) in the kernel; normed is then only written (and returned) when
    final."""
    _lib.require_cuda(x, mix, gate, shift, scale, norm_w, residual, rowmap, path_scale)
    if (x is None) != (x_from is not None) or (x_from is not None and (residual is None or path_scale is not None or mix_bcast)):
        raise RuntimeError("block_tail: x_from replaces x, needs the residual and takes no path_scale / mix_bcast")
    if x_from is not None:
        x_rstd, x_norm_w = x_from
        _lib.require_cuda(x_rstd, x_norm_w)
        xdt, xdev = x_norm_w.dtype, residual.device
        Bt, L, D = residual.shape
        if x_rstd.dtype != torch.float32 or x_rstd.numel() != Bt * L or not x_rstd.is_contiguous() or x_norm_w.numel() != D:
            raise RuntimeError("block_tail: x_from needs the previous tail's (Bt * L,) fp32 rstd and its (D,) norm_w")
    else:
        xdt, xdev = x.dtype, x.device
        Bt, L, D = x.shape
    if path_scale is not None and (path_scale.dtype != xdt or tuple(path_scale.shape) != (Bt,) or not path_scale.is_contiguous()):
        raise RuntimeError(f"block_tail: path_scale must be a contiguous ({Bt},) tensor in {xdt}, got "
                           f"{tuple(path_scale.shape)} {path_scale.dtype}")
    if mod_div != 1:
        # modulation vectors are per ORIGINAL batch element; expand to the folded batch (tiny)
        gate = None if gate is None else gate.repeat_interleave(mod_div, dim=0)
        shift = None if shift is None else shift.repeat_interleave(mod_div, dim=0)
        scale = None if scale is None else scale.repeat_interleave(mod_div, dim=0)
    mods = [m for m in (gate, shift, scale) if m is not None]
    rs = mods[0].stride(0) if mods else 0
    for m in mods:
        if m.stride(0) != rs or m.stride(1) != 1:
            raise RuntimeError("block_tail: modulation views must share one row stride")
    if norm_w.dtype != xdt:
        norm_w = norm_w.to(xdt)
    # the kernel reads every operand with ONE dtype (x's).  Under bf16 autocast with fp32 master weights the tokens can be
    # fp32 (embed() adds an fp32 pos_embed) while the adaLN chunks and the mixer output are bf16: bring them to x.dtype
    # instead of letting the kernel reinterpret the buffers.
    def _as_x(t):
        return t if (t is None or t.dtype == xdt) else t.to(xdt)
    mix = _as_x(mix)
    if mix is not None and not mix.is_contiguous():
        mix = mix.contiguous()
    if any(m is not None and m.dtype != xdt for m in (gate, shift, scale)):
        # re-materialise the three views in x.dtype with one common row stride
        D_ = D
        packed = torch.zeros((Bt // mod_div if mod_div != 1 else Bt, 3 * D_), dtype=xdt, device=xdev)
        for i_, m in enumerate((gate, shift, scale)):
            if m is not None:
                packed[:, i_ * D_:(i_ + 1) * D_] = m
        gate = None if gate is None else packed[:, :D_]
        shift = None if shift is None else packed[:, D_:2 * D_]
        scale = None if scale is None else packed[:, 2 * D_:]
    if residual is not None and residual.dtype != torch.float32:
        raise RuntimeError("block_tail: the residual stream must be fp32 (residual_in_fp32=True)")
    res_out = torch.empty((Bt, L, D), dtype=torch.float32, device=xdev) if not final else None
    normed = torch.empty((Bt, L, D), dtype=xdt, device=xdev) if (x_from is None or final) else None
    modded = torch.empty((Bt, L, D), dtype=xdt, device=xdev) if (want_modded and not final) else None
    p = _lib.BlockTailParams()
    p.x, p.mix, p.gate, p.shift, p.scale = _lib.ptr(x), _lib.ptr(mix), _lib.ptr(gate), _lib.ptr(shift), _lib.ptr(scale)
    p.norm_w, p.residual, p.rowmap = _lib.ptr(norm_w), _lib.ptr(residual), _lib.ptr(rowmap)
    p.residual_out, p.normed, p.modded = _lib.ptr(res_out), _lib.ptr(normed), _lib.ptr(modded)
    p.mod_rs = rs
    p.batch, p.seqlen, p.dim = Bt, L, D
    p.dtype, p.final_layer, p.eps = _lib.dt(xdt), int(final), float(eps)
    rstd = torch.empty((Bt * L,), dtype=torch.float32, device=xdev) if want_rstd else None
    p.rstd = _lib.ptr(rstd)
    if mix_bcast and (mix is None or mix.numel() != L * D or gate is not None or rowmap is not None or residual is not None):
        raise RuntimeError("block_tail: mix_bcast takes a (seqlen, dim) mix table and no gate / rowmap / residual")
    if x_from is not None:
        _lib.call("zg_block_tail_fwd_rebuild", _lib.BlockTailRebuildParams(p, _lib.ptr(x_rstd), _lib.ptr(x_norm_w)))
    elif path_scale is not None:
        _lib.call("zg_block_tail_fwd_dp", _lib.BlockTailDpParams(p, _lib.ptr(path_scale)))
    else:
        _lib.call("zg_block_tail_fwd_pe" if mix_bcast else "zg_block_tail_fwd", p)
    if want_rstd:
        return res_out, normed, modded, rstd
    return res_out, normed, modded


def text_prologue(x, mix, gate, shift, scale, rowmap, eps, mod_div=1, want_stats=False):
    """zg_text_prologue_fwd wrapper, the text branch of a has_text block up to the attention (model_zigma.py:206-208):
    hidden = x + gate * mix[:, rowmap];  q_in = modulate(LayerNorm_noaffine(hidden, eps), shift, scale).
    x, mix: (Bt, L, D) contiguous in one dtype; rowmap: int32 (L,) or None; gate / shift / scale: (Bt // mod_div, D) views in
    that dtype with a common row stride.  Returns hidden, q_in (and the fp32 (Bt * L,) mean, rstd when want_stats)."""
    _lib.require_cuda(x, mix, gate, shift, scale, rowmap)
    Bt, L, D = x.shape
    if mod_div != 1:
        # modulation vectors are per ORIGINAL batch element; expand to the folded batch (tiny), as block_tail does
        gate, shift, scale = (m.repeat_interleave(mod_div, dim=0) for m in (gate, shift, scale))
    if any(t.dtype != x.dtype for t in (mix, gate, shift, scale)) or tuple(mix.shape) != (Bt, L, D) or not mix.is_contiguous():
        raise RuntimeError("text_prologue: mix must be a contiguous tensor of x's shape and every operand in x's dtype")
    rs = gate.stride(0)
    if any(m.stride(0) != rs or m.stride(1) != 1 or tuple(m.shape) != (Bt, D) for m in (gate, shift, scale)):
        raise RuntimeError("text_prologue: gate / shift / scale must be (batch, dim) views sharing one row stride")
    hidden, q_in = torch.empty_like(x), torch.empty_like(x)
    mean = torch.empty((Bt * L,), dtype=torch.float32, device=x.device) if want_stats else None
    rstd = torch.empty((Bt * L,), dtype=torch.float32, device=x.device) if want_stats else None
    p = _lib.TextPrologueParams()
    p.x, p.mix, p.gate, p.shift, p.scale, p.rowmap = _lib.ptr(x), _lib.ptr(mix), _lib.ptr(gate), _lib.ptr(shift), _lib.ptr(scale), _lib.ptr(rowmap)
    p.hidden, p.q_in, p.mean, p.rstd = _lib.ptr(hidden), _lib.ptr(q_in), _lib.ptr(mean), _lib.ptr(rstd)
    p.mod_rs = rs
    p.batch, p.seqlen, p.dim, p.dtype, p.eps = Bt, L, D, _lib.dt(x), float(eps)
    _lib.call("zg_text_prologue_fwd", p)
    if want_stats:
        return hidden, q_in, mean, rstd
    return hidden, q_in


class ZigMaEngine:
    def __init__(self, model):
        self.m = model
        self._versions = None
        self._graphs = {}
        self.use_graph = os.environ.get("ZIGMA_CUDA_GRAPH", "1") != "0"
        # dt_proj inside the scan kernel (zg_scan_params.dt_w): correct and tested, but off by default (not measured on H100; it was slower than GEMM + scan where it was last measured)
        # (0.600 ms vs 0.507 + 0.042 ms per layer at config 2: the MMA + fragment epilogue lengthens the latency-bound
        # pre phase of every stage), so it is opt-in
        self.fuse_dt = os.environ.get("ZIGMA_FUSE_DT", "0") == "1"
        self.refresh()

    # ---- derived, cached tensors ------------------------------------------------------------------
    def _param_versions(self):
        return tuple((p.data_ptr(), p._version) for p in self.m.parameters())

    def refresh(self):
        m = self.m
        dev = next(m.parameters()).device
        self.layers = []
        for blk in m.blocks:
            mx = blk.mixer
            E, W = mx.d_inner, mx.d_conv

            def pack(sfx=""):
                conv, xp, dp = getattr(mx, "conv1d" + sfx), getattr(mx, "x_proj" + sfx), getattr(mx, "dt_proj" + sfx)
                A_log = mx.A_b_log if sfx else mx.A_log
                Dp = mx.D_b if sfx else mx.D
                return dict(conv_w=conv.weight.detach().reshape(E, W).contiguous(),
                            conv_b=None if conv.bias is None else conv.bias.detach().contiguous(),
                            x_proj=xp.weight.detach(), dt_proj=dp.weight.detach(),
                            A=(-torch.exp(A_log.detach().float())).contiguous(), D=Dp.detach().float().contiguous(),
                            dt_bias=dp.bias.detach().float().contiguous())
            L = dict(fwd=pack(), in_proj=mx.in_proj.weight.detach(), in_bias=None if mx.in_proj.bias is None else mx.in_proj.bias.detach(),
                     out_proj=mx.out_proj.weight.detach(), out_bias=None if mx.out_proj.bias is None else mx.out_proj.bias.detach(),
                     norm_w=blk.norm.weight.detach(), R=mx.dt_rank, N=mx.d_state, E=E, st=mx.scan_type)
            if mx.scan_type == "v2":
                L["bwd"] = pack("_b")
            if mx.zigzag_paths is not None:
                L["perm"] = _i32(mx.zigzag_paths[mx.layer_idx].to(dev))
                L["perm_rev"] = _i32(mx.zigzag_paths_reverse[mx.layer_idx].to(dev))
                L["perm64"] = mx.zigzag_paths[mx.layer_idx].to(dev)
                L["perm_rev64"] = mx.zigzag_paths_reverse[mx.layer_idx].to(dev)
            if mx.st_order is not None:
                L["s_or_t"] = mx.st_order[mx.layer_idx]
            self.layers.append(L)
        # every block's adaLN Linear in ONE GEMM: (B, D) @ (D, depth * 3D)
        self.ada_w = torch.cat([b.adaLN_modulation[1].weight.detach() for b in m.blocks], dim=0).contiguous()
        self.ada_b = torch.cat([b.adaLN_modulation[1].bias.detach() for b in m.blocks], dim=0).contiguous()
        self._rev_cache = {}
        self._pe_w = None                       # zero-padded patch-embedding weight (bf16), built on first use
        self._versions = self._param_versions()
        self._graphs = {}

    def _flip_map(self, L, dev):
        if L not in self._rev_cache:
            self._rev_cache[L] = torch.arange(L - 1, -1, -1, dtype=torch.int32, device=dev)
        return self._rev_cache[L]

    # ---- one directional pass of the mixer core, token major ------------------------------------------
    def _core(self, xz, Bt, L, lay, w, rowmap, acc_into=None):
        """xz: (Bt*L, 2E) token-major.  Returns y (Bt, L, E) = scan(...) * silu(z), in scan order.  acc_into: (Bt, L, E) result of
        the forward sweep -- this (backward) sweep is written flipped and added into it by the scan kernel itself."""
        E, R, N = lay["E"], lay["R"], lay["N"]
        xz3 = xz.view(Bt, L, 2 * E)
        x_log = xz3[:, :, :E].transpose(1, 2)          # logical (Bt, E, L), dim-contiguous
        z_log = xz3[:, :, E:].transpose(1, 2)
        xc = _conv_fwd(x_log, w["conv_w"], w["conv_b"], True, x_rowmap=rowmap)           # logical (Bt, E, L), token-major memory
        xc_flat = xc.transpose(1, 2).reshape(Bt * L, E)
        x_dbl = _linear(xc_flat, w["x_proj"])                                              # (Bt*L, R + 2N)
        xd3 = x_dbl.view(Bt, L, R + 2 * N)
        B_log = xd3[:, :, R:R + N].permute(0, 2, 1).unsqueeze(1)                           # (Bt, 1, N, L) view
        C_log = xd3[:, :, R + N:].permute(0, 2, 1).unsqueeze(1)
        extra = {} if acc_into is None else dict(out=acc_into.transpose(1, 2), out_reverse=True, out_accumulate=True)
        if self.fuse_dt and fused_dt_ok(xz.dtype, E, L, N, R, w["dt_proj"]):
            # dt_proj inside the scan kernel (tensor-core prologue): no delta tensor, no dt_proj GEMM launch
            y, _, _, _ = _scan_fwd(xc, None, w["A"], B_log, C_log, w["D"], z_log, w["dt_bias"], True,
                                   z_rowmap=rowmap, want_last_state=False, want_ckpt=False, dt_proj=(w["dt_proj"], xd3), **extra)
        else:
            delta = _linear(x_dbl[:, :R], w["dt_proj"])                                    # (Bt*L, E)
            d_log = delta.view(Bt, L, E).transpose(1, 2)
            y, _, _, _ = _scan_fwd(xc, d_log, w["A"], B_log, C_log, w["D"], z_log, w["dt_bias"], True,
                                   z_rowmap=rowmap, want_last_state=False, want_ckpt=False, **extra)
        return y.transpose(1, 2)                                                            # (Bt, L, E) contiguous

    def _patch_embed(self, x):
        """Patch embedding (model_zigma.py:608-614: a Conv2d with kernel = stride = patch, i.e. a per-patch linear map) as a GEMM
        on the wgmma kernel: the K = C p^2 columns (4 at patch 1) are zero-padded to the 16-byte row pitch TMA needs.  Returns
        (B, L, D) tokens, or None when the model is not bf16 (the module's own forward runs then)."""
        m = self.m
        if x.dtype != torch.bfloat16 or os.environ.get("ZIGMA_TCGEN05", "1") != "1":
            return None
        emb = m.x_embedder
        p = emb.patch_size[0]
        lead = x.shape[:-3]
        x4 = x.reshape(-1, *x.shape[-3:])                    # video: (B T, C, H, W)
        Bn, C, H, W = x4.shape
        if p == 1:
            tok = x4.flatten(2).transpose(1, 2)
        else:
            tok = x4.reshape(Bn, C, H // p, p, W // p, p).permute(0, 2, 4, 1, 3, 5).reshape(Bn, (H // p) * (W // p), C * p * p)
        K = tok.shape[-1]
        if self._pe_w is None:
            Kp = (K + 7) // 8 * 8
            w = torch.zeros((emb.proj.weight.shape[0], Kp), dtype=torch.bfloat16, device=x.device)
            w[:, :K] = emb.proj.weight.detach().reshape(w.shape[0], -1)
            self._pe_w = w
        Kp = self._pe_w.shape[1]
        tp = torch.zeros((tok.shape[0] * tok.shape[1], Kp), dtype=torch.bfloat16, device=x.device)
        tp[:, :K] = tok.reshape(-1, K)
        out = _linear(tp, self._pe_w, None if emb.proj.bias is None else emb.proj.bias.detach())
        return out.view(*lead[:1], -1, out.shape[-1]) if len(lead) == 2 else out.view(Bn, -1, out.shape[-1])

    def _temporal_fused_ok(self, dtype, lay, T, K):
        E, N = lay["E"], lay["N"]
        return (scan_hot_path_ok(dtype, E, T, N, lay["R"]) and (T * K) % 32 == 0
                and os.environ.get("ZIGMA_TEMPORAL_FUSED", "1") != "0" and not self.fuse_dt)

    def _temporal_tables(self, lay, T, K, dev):
        """Composite row tables of a temporal layer (int32, length T K): position p = k T + t of the (k, t)-ordered working layout
        <-> token (perm[t], k) of the (t, k)-ordered model layout."""
        key = ("temporal", id(lay), T, K)
        if key not in self._rev_cache:
            perm, rev = lay["perm64"], lay["perm_rev64"]
            k = torch.arange(K, device=dev)
            comp_in = (perm.view(1, T) * K + k.view(K, 1)).reshape(-1)                    # [k T + t] -> perm[t] K + k
            comp_out = (k.view(1, K) * T + rev.view(T, 1)).reshape(-1)                    # [t K + k] -> k T + perm_rev[t]
            self._rev_cache[key] = {"in": comp_in.to(torch.int32).contiguous(), "out": comp_out.to(torch.int32).contiguous()}
        return self._rev_cache[key]

    def _core_temporal(self, xz, B, T, K, lay, w, tb):
        """Temporal layer of a factorised video scan (mamba_simple.py:416-442) on the (B T K, 2E) token-major xz, no permuted
        copies.  Returns y (B K T, E) in (b, k, t) order."""
        E, R, N = lay["E"], lay["R"], lay["N"]
        L = T * K
        xz3 = xz.view(B, L, 2 * E)
        x_log = xz3[:, :, :E].transpose(1, 2)                                              # logical (B, E, L), dim-contiguous
        xc = _conv_fwd(x_log, w["conv_w"], w["conv_b"], True, x_rowmap=tb["in"], seg_len=T)   # (B, L, E) memory, (k, t) order
        xc_flat = xc.transpose(1, 2).reshape(B * L, E)
        x_dbl = _linear(xc_flat, w["x_proj"])
        delta = _linear(x_dbl[:, :R], w["dt_proj"])
        u_log = xc_flat.view(B * K, T, E).transpose(1, 2)
        d_log = delta.view(B * K, T, E).transpose(1, 2)
        xd3 = x_dbl.view(B * K, T, R + 2 * N)
        B_log = xd3[:, :, R:R + N].permute(0, 2, 1).unsqueeze(1)
        C_log = xd3[:, :, R + N:].permute(0, 2, 1).unsqueeze(1)
        z_btk = xz.view(B, T, K, 2 * E)[:, :, :, E:]                                       # (B, T, K, E) strided view of the z half
        y, _, _, _ = _scan_fwd(u_log, d_log, w["A"], B_log, C_log, w["D"], None, w["dt_bias"], True, z_rowmap=lay["perm"],
                               want_last_state=False, want_ckpt=False, z_btk=z_btk)
        return y.transpose(1, 2)

    def _mixer(self, modded, lay):
        """modded: (B, L, D) -> (mix (Bt', L', D) token-major in SCAN order, tail rowmap, fold info)."""
        B, L, D = modded.shape
        E = lay["E"]
        xz = _linear(modded.reshape(B * L, D), lay["in_proj"], lay["in_bias"])
        st = lay["st"]
        if st == "v1":
            y = self._core(xz, B, L, lay, lay["fwd"], None)
            rowmap = None
        elif st == "v2":
            yf = self._core(xz, B, L, lay, lay["fwd"], None)
            if scan_hot_path_ok(xz.dtype, E, L, lay["N"], lay["R"]):
                # y = yf + yb.flip(1) inside the second scan (ZG_SCAN_OUT_REVERSE | ZG_SCAN_OUT_ACCUMULATE): no flipped copy, no add kernel
                y = self._core(xz, B, L, lay, lay["bwd"], self._flip_map(L, xz.device), acc_into=yf)
            else:
                yb = self._core(xz, B, L, lay, lay["bwd"], self._flip_map(L, xz.device))
                y = yf + yb.flip(1)
            rowmap = None
        elif "s_or_t" not in lay:
            y = self._core(xz, B, L, lay, lay["fwd"], lay["perm"])
            rowmap = lay["perm_rev"]
        else:
            T = self.m.video_frames
            K = L // T
            if lay["s_or_t"] == "s":      # (b t) sequences of K tokens: a pure re-view of token-major memory
                y = self._core(xz, B * T, K, lay, lay["fwd"], lay["perm"])
                mix = _linear(y.reshape(B * T * K, E), lay["out_proj"], lay["out_bias"]).view(B * T, K, D)
                return mix, lay["perm_rev"], T
            # (b k) sequences of T tokens: strided in the (b, t k) token-major memory
            if self._temporal_fused_ok(xz.dtype, lay, T, K):
                # no copies: the conv gathers its input rows through a composite table (segments of T positions), the scan
                # reads z through a two-level batch, and the block tail un-permutes with the inverse composite table
                tb = self._temporal_tables(lay, T, K, xz.device)
                y = self._core_temporal(xz, B, T, K, lay, lay["fwd"], tb)
                mix = _linear(y.reshape(B * L, E), lay["out_proj"], lay["out_bias"]).view(B, L, D)        # rows in (b, k, t) order
                return mix, tb["out"], 1
            xz_t = xz.view(B, T, K, 2 * E).permute(0, 2, 1, 3).reshape(B * K * T, 2 * E)
            y = self._core(xz_t, B * K, T, lay, lay["fwd"], lay["perm"])
            mix = _linear(y.reshape(B * K * T, E), lay["out_proj"], lay["out_bias"]).view(B * K, T, D)
            mix = mix[:, lay["perm_rev64"], :].reshape(B, K, T, D).permute(0, 2, 1, 3).reshape(B, L, D)
            return mix, None, 1
        mix = _linear(y.reshape(B * L, E), lay["out_proj"], lay["out_bias"]).view(B, L, D)
        return mix, rowmap, 1

    # ---- whole forward -----------------------------------------------------------------------------
    def _forward_impl(self, x, t, y):
        m = self.m
        tokens = self._patch_embed(x)
        # `tokens + pos_embed` (model_zigma.py:941) inside the first tail (mix = the (L, D) table, no gate) instead of an
        # elementwise pass of its own: same rounding (one add in the token dtype).  Not with a temporal embedding on top.
        pe = None
        if (tokens is not None and m.use_pe in (1, 2) and not (m.video_frames > 0 and m.tpe) and m.pos_embed.dtype == tokens.dtype
                and tokens.shape[-1] <= 2048 and os.environ.get("ZIGMA_FOLD_PE", "1") != "0"):
            pe = m.pos_embed.detach().reshape(-1, m.pos_embed.shape[-1]).contiguous()
        hs, c, text = m.embed(x, t, y, tokens=tokens, add_pos=pe is None)
        hs = hs.contiguous()
        B, L, D = hs.shape
        if pe is not None and pe.shape[0] != L:
            raise RuntimeError(f"pos_embed has {pe.shape[0]} rows, the model {L} tokens")
        depth = len(self.layers)
        nmod = 6 if m.has_text else 3          # (+ shift, scale, gate of the text cross-attention branch)
        mods = _linear(F.silu(c), self.ada_w, self.ada_b).view(B, depth, nmod, D)  # shift, scale, gate per block (one GEMM for all)
        eps = m.blocks[0].norm.eps
        lay0 = self.layers[0]
        # below the first tail, each tail rebuilds its x (the previous tail's normed output) from the residual row it reads anyway
        # and the previous tail's rstd and norm_w, so normed is not written and read back between tails.  Not for text blocks:
        # their prologue reads normed.
        rebuild = not m.has_text and D <= 1024
        residual, normed, modded, *rstd = block_tail(hs, pe, None, mods[:, 0, 0], mods[:, 0, 1], lay0["norm_w"], None, None, eps,
                                                     mix_bcast=pe is not None, want_rstd=rebuild)
        prev_w = lay0["norm_w"]
        for i, lay in enumerate(self.layers):
            mix, rowmap, fold = self._mixer(modded, lay)
            last = i == depth - 1
            nw = m.norm_f.weight if last else self.layers[i + 1]["norm_w"]
            neps = m.norm_f.eps if last else m.blocks[i + 1].norm.eps
            gate = mods[:, i, 2]
            shift = None if last else mods[:, i + 1, 0]
            scale = None if last else mods[:, i + 1, 1]
            if m.has_text:
                # text blocks (model_zigma.py:446-458): the mixer's gated residual has to exist before the cross-attention
                # reads it; the attention branch (zg_cross_attn_fwd on the text tokens) then takes the place of the mixer output
                # in the fused tail:  hidden2 = hidden + gate_msa * msa(modulate(norm_msa(hidden)))
                blk = m.blocks[i]
                # one kernel un-permutes the mixer output with the layer's own row table -- (B fold, L / fold) rows for a spatial
                # video layer (same memory as (B, L)), the composite (k T + t) table of a copy-free temporal layer, the zigzag
                # table otherwise -- and forms hidden and the attention's query input
                Bf = B * fold
                hidden, q_in = text_prologue(normed.view(Bf, L // fold, D), mix.view(Bf, L // fold, D), gate, mods[:, i, 3], mods[:, i, 4],
                                             rowmap, blk.norm_msa.eps, mod_div=fold)
                fold = 1
                mix, rowmap, gate, normed = blk.msa(q_in.view(B, L, D), text=text, mask=None).contiguous(), None, mods[:, i, 5], hidden.view(B, L, D)
            tail_x = dict(x_from=(rstd[0], prev_w.to(hs.dtype)), want_rstd=not last) if rebuild else {}
            if fold != 1:     # spatial video layer: rows are (b t, k); same memory as (b, t k)
                Bf = B * fold
                residual, normed, modded, *rstd = block_tail(None if rebuild else normed.view(Bf, L // fold, D), mix, gate, shift, scale,
                                                             nw, residual.view(Bf, L // fold, D), rowmap, neps, final=last, mod_div=fold,
                                                             **tail_x)
                normed = normed.view(B, L, D) if normed is not None else None
                if not last:
                    residual, modded = residual.view(B, L, D), modded.view(B, L, D)
            else:
                residual, normed, modded, *rstd = block_tail(None if rebuild else normed, mix, gate, shift, scale, nw, residual, rowmap,
                                                             neps, final=last, **tail_x)
            prev_w = nw
        out = _linear(normed.reshape(B * L, D), m.final_layer.linear.weight, m.final_layer.linear.bias).view(B, L, -1)   # un-embed
        if m.video_frames > 0:
            return m.unpatchify_video(out, m.video_frames)
        return m.unpatchify(out)

    @torch.no_grad()
    def forward(self, x, t, y=None):
        if self._versions != self._param_versions():
            self.refresh()
        if not self.use_graph:
            return self._forward_impl(x, t, y)
        key = (tuple(x.shape), x.dtype, tuple(t.shape), t.dtype, None if y is None else (tuple(y.shape), y.dtype))
        g = self._graphs.get(key)
        if g is None:
            # warm-up on a side stream (sets kernel attributes, fills cuBLAS workspaces), then capture
            sx, st_, sy = x.clone(), t.clone(), None if y is None else y.clone()
            s = torch.cuda.Stream()
            s.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(s):
                for _ in range(2):
                    self._forward_impl(sx, st_, sy)
            torch.cuda.current_stream().wait_stream(s)
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph):
                sout = self._forward_impl(sx, st_, sy)
            g = (graph, sx, st_, sy, sout)
            self._graphs[key] = g
        graph, sx, st_, sy, sout = g
        sx.copy_(x)
        st_.copy_(t)
        if y is not None:
            sy.copy_(y)
        graph.replay()
        return sout.clone()

    @torch.no_grad()
    def sample_euler(self, x0, ts, y=None, return_trajectory=False, dts=None):
        """Fixed-grid Euler integration x_{i+1} = x_i + (t_{i+1} - t_i) * model(x_i, t_i) over the grid ``ts`` -- what
        ``Sampler.sample_ode(sampling_method="euler")`` makes torchdiffeq do for a velocity model on the linear path
        (transport/integrators.py:105-123, transport.py:372-417) -- with the WHOLE loop captured as one CUDA graph: the
        time vector is filled in-graph (one fill per step with the step's constant), the update runs in-graph, nothing is
        copied or cloned between the steps.  Returns the final state (or the (len(ts), ...) trajectory)."""
        if self._versions != self._param_versions():
            self.refresh()
        ts = [float(v) for v in ts]
        dts = [b - a for a, b in zip(ts, ts[1:])] if dts is None else [float(v) for v in dts]   # (fp32 differences of an fp32 grid, if given)
        key = ("euler", tuple(x0.shape), x0.dtype, tuple(ts), tuple(dts), None if y is None else (tuple(y.shape), y.dtype), bool(return_trajectory))
        g = self._graphs.get(key)
        if g is None:
            sx, sy = x0.clone(), None if y is None else y.clone()
            tvec = torch.empty(x0.shape[0], device=x0.device, dtype=x0.dtype)

            def loop():
                x, traj = sx, [sx]
                for t0, dt in zip(ts, dts):
                    tvec.fill_(t0)
                    x = torch.add(x, self._forward_impl(x, tvec, sy), alpha=dt)
                    if return_trajectory:
                        traj.append(x)
                return torch.stack(traj, 0) if return_trajectory else x
            if not self.use_graph:
                return loop_eager(self, x0, ts, dts, y, return_trajectory)
            s = torch.cuda.Stream()
            s.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(s):
                tvec.fill_(ts[0])
                for _ in range(2):
                    self._forward_impl(sx, tvec, sy)          # warm-up: kernel attributes, workspaces
            torch.cuda.current_stream().wait_stream(s)
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph):
                sout = loop()
            g = (graph, sx, sy, sout)
            self._graphs[key] = g
        graph, sx, sy, sout = g
        sx.copy_(x0)
        if y is not None:
            sy.copy_(y)
        graph.replay()
        return sout.clone()


def loop_eager(engine, x0, ts, dts, y, return_trajectory):
    x, traj = x0, [x0]
    tvec = torch.empty(x0.shape[0], device=x0.device, dtype=x0.dtype)
    for t0, dt in zip(ts, dts):
        tvec.fill_(t0)
        x = torch.add(x, engine._forward_impl(x, tvec, y), alpha=dt)
        if return_trajectory:
            traj.append(x)
    return torch.stack(traj, 0) if return_trajectory else x
