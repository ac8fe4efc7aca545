"""ZigMa denoiser (``model_zigma.py`` of the reference) on the sm_90a kernels.

Keeps the ``ZigMa(...)`` constructor (:549-576), ``forward(hidden_states, t, y=None)`` (:911-916) and
the state-dict key layout (SURVEY.md section 8b) so reference checkpoints load unchanged.  Under
``torch.no_grad()`` / eval the forward is executed by ``engine.ZigMaEngine`` (token-major fused
kernels, CUDA-graph capturable); with autograd enabled it runs module by module through the op
interfaces (``rms_norm_fn``, ``mamba_inner_fn`` ...) exactly like the reference's Block.forward.
"""
import math
from functools import partial

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

from .layernorm import RMSNorm, layer_norm_fn, rms_norm_fn
from .mamba_simple import Mamba
from .utils_zigzag import hilbert_path, reverse_permut_np, zigzag_path


_FREQ_CACHE = {}


def modulate(x, shift, scale):
    return x * (1 + scale.unsqueeze(1)) + shift.unsqueeze(1)


class PatchEmbed(nn.Module):
    """2-D latent -> tokens: Conv2d(kernel = stride = patch) + flatten + transpose.  Stands in for
    timm.models.vision_transformer.PatchEmbed (third party, unpinned; model_zigma.py:17,608-614) with
    the attributes the reference touches: .proj, .patch_size, .num_patches."""

    def __init__(self, img_size, patch_size, in_chans, embed_dim, bias=True):
        super().__init__()
        self.img_size = (img_size, img_size)
        self.patch_size = (patch_size, patch_size)
        self.grid_size = (img_size // patch_size, img_size // patch_size)
        self.num_patches = self.grid_size[0] * self.grid_size[1]
        self.proj = nn.Conv2d(in_chans, embed_dim, kernel_size=patch_size, stride=patch_size, bias=bias)

    def forward(self, x):
        # kernel == stride: the strided Conv2d is a per-patch linear map.  Done as unfold + GEMM so the
        # fp32 path stays exact fp32 (cuDNN convolutions default to TF32: torch.backends.cudnn.allow_tf32)
        # and the bf16 path goes through the same library GEMM as every other projection.
        B, C, H, W = x.shape
        p = self.patch_size[0]
        if p == 1:
            tokens = x.flatten(2).transpose(1, 2)                                   # (B, H*W, C)
        else:
            tokens = (x.reshape(B, C, H // p, p, W // p, p).permute(0, 2, 4, 1, 3, 5).reshape(B, (H // p) * (W // p), C * p * p))
        return F.linear(tokens, self.proj.weight.reshape(self.proj.weight.shape[0], -1), self.proj.bias)


class PatchEmbed_Video(PatchEmbed):
    """(B, T, C, H, W) -> (B, T*N, D).  model_zigma.py:66-78."""

    def forward(self, x):
        B, T = x.shape[:2]
        x = super().forward(x.reshape(B * T, *x.shape[2:]))
        return x.reshape(B, T * x.shape[1], x.shape[2])


class CrossAttention(nn.Module):
    """Text cross-attention of has_text blocks (model_zigma.py:95-135); library SDPA, not on the
    benchmarked path (none of the BASELINE configs sets has_text)."""

    def __init__(self, query_dim, context_dim=None, heads=8, dim_head=64, dropout=0.0):
        super().__init__()
        inner = dim_head * heads
        context_dim = query_dim if context_dim is None else context_dim
        self.heads = heads
        self.to_q = nn.Linear(query_dim, inner, bias=False)
        self.to_k = nn.Linear(context_dim, inner, bias=False)
        self.to_v = nn.Linear(context_dim, inner, bias=False)
        self.to_out = nn.Sequential(nn.Linear(inner, query_dim), nn.Dropout(dropout))

    def forward(self, x, text, mask=None):
        B = x.shape[0]
        split = lambda t: t.reshape(B, t.shape[1], self.heads, -1).transpose(1, 2)
        o = F.scaled_dot_product_attention(split(self.to_q(x)), split(self.to_k(text)), split(self.to_v(text)))
        return self.to_out(o.transpose(1, 2).reshape(B, x.shape[1], -1))


class DropPath(nn.Module):
    """Stochastic depth per sample (model_zigma.py:138-174)."""

    def __init__(self, drop_prob=0.0, scale_by_keep=True):
        super().__init__()
        self.drop_prob, self.scale_by_keep = drop_prob, scale_by_keep

    def forward(self, x):
        if self.drop_prob == 0.0 or not self.training:
            return x
        keep = 1 - self.drop_prob
        mask = x.new_empty((x.shape[0],) + (1,) * (x.ndim - 1)).bernoulli_(keep)
        if keep > 0.0 and self.scale_by_keep:
            mask.div_(keep)
        return x * mask


class TimestepEmbedder(nn.Module):
    """Sinusoid(256) -> Linear -> SiLU -> Linear (model_zigma.py:232-275).  The frequency table is
    computed in the MODEL dtype as in the reference (:259-261)."""

    def __init__(self, hidden_size, dtype, frequency_embedding_size=256):
        super().__init__()
        self.mlp = nn.Sequential(nn.Linear(frequency_embedding_size, hidden_size, bias=True), nn.SiLU(),
                                 nn.Linear(hidden_size, hidden_size, bias=True))
        self.dtype = dtype
        self.frequency_embedding_size = frequency_embedding_size

    @staticmethod
    def timestep_embedding(t, dim, dtype, max_period=10000):
        half = dim // 2
        key = (dim, dtype, t.device, max_period)
        freqs = _FREQ_CACHE.get(key)
        if freqs is None:   # computed on the host in the model dtype exactly as the reference does, then cached
            freqs = torch.exp(-math.log(max_period) * torch.arange(start=0, end=half, dtype=dtype) / half).to(device=t.device)
            _FREQ_CACHE[key] = freqs   # (a per-call H2D copy would also break CUDA-graph capture)
        args = t[:, None].float() * freqs[None]
        emb = torch.cat([torch.cos(args), torch.sin(args)], dim=-1)
        if dim % 2:
            emb = torch.cat([emb, torch.zeros_like(emb[:, :1])], dim=-1)
        return emb

    def forward(self, t):
        return self.mlp(self.timestep_embedding(t, self.frequency_embedding_size, dtype=self.dtype).to(dtype=self.dtype))


class LabelEmbedder(nn.Module):
    """Class-label table with optional CFG dropout row (model_zigma.py:278-310)."""

    def __init__(self, num_classes, hidden_size, dropout_prob):
        super().__init__()
        self.embedding_table = nn.Embedding(num_classes + int(dropout_prob > 0), hidden_size)
        self.num_classes, self.dropout_prob = num_classes, dropout_prob

    def forward(self, labels, train, force_drop_ids=None):
        if (train and self.dropout_prob > 0) or force_drop_ids is not None:
            drop = (torch.rand(labels.shape[0], device=labels.device) < self.dropout_prob) if force_drop_ids is None else (force_drop_ids == 1)
            labels = torch.where(drop, self.num_classes, labels)
        return self.embedding_table(labels)


class FinalLayer(nn.Module):
    """LayerNorm(no affine, eps 1e-6) -> Linear(D, p*p*C) (model_zigma.py:313-337)."""

    def __init__(self, hidden_size, patch_size, out_channels, cond=False):
        super().__init__()
        self.norm_final = nn.LayerNorm(hidden_size, elementwise_affine=False, eps=1e-6)
        self.linear = nn.Linear(hidden_size, patch_size * patch_size * out_channels, bias=True)
        if cond:
            self.adaLN_modulation = nn.Sequential(nn.SiLU(), nn.Linear(hidden_size, 2 * hidden_size, bias=True))

    def forward(self, x, c=None):
        if c is not None:
            shift, scale = self.adaLN_modulation(c).chunk(2, dim=1)
            return self.linear(modulate(self.norm_final(x), shift, scale))
        return self.linear(self.norm_final(x))


class Block(nn.Module):
    """Add -> Norm -> adaLN-modulated Mamba mixer (-> text cross-attention).  model_zigma.py:340-460."""

    def __init__(self, dim, mixer_cls, has_text=False, norm_cls=nn.LayerNorm, fused_add_norm=False,
                 residual_in_fp32=False, drop_path=0.0, skip=False):
        super().__init__()
        self.residual_in_fp32 = residual_in_fp32
        self.fused_add_norm = fused_add_norm
        self.has_text = has_text
        self.mixer = mixer_cls(dim)
        self.norm = norm_cls(dim)
        self.drop_path = DropPath(drop_path) if drop_path > 0.0 else nn.Identity()
        if fused_add_norm:
            assert isinstance(self.norm, (nn.LayerNorm, RMSNorm)), "Only LayerNorm and RMSNorm are supported for fused_add_norm"
        self.skip_linear = nn.Linear(2 * dim, dim) if skip else None
        self.adaLN_modulation = nn.Sequential(nn.SiLU(), nn.Linear(dim, (6 if has_text else 3) * dim, bias=True))
        if has_text:
            self.msa = CrossAttention(query_dim=dim, context_dim=dim, heads=8, dim_head=64, dropout=0.0)
            self.norm_msa = nn.LayerNorm(dim, elementwise_affine=False, eps=1e-6)

    def forward(self, x, residual=None, c=None, text=None, inference_params=None, skip=None):
        if self.skip_linear is not None:
            x = self.skip_linear(torch.cat([x, skip], dim=-1))
        if not self.fused_add_norm:
            residual = x if residual is None else residual + self.drop_path(x)
            x = self.norm(residual.to(dtype=self.norm.weight.dtype))
            if self.residual_in_fp32:
                residual = residual.to(torch.float32)
        else:
            fn = rms_norm_fn if isinstance(self.norm, RMSNorm) else layer_norm_fn
            x, residual = fn(x if residual is None else self.drop_path(x), self.norm.weight, self.norm.bias,
                             residual=residual, prenorm=True, residual_in_fp32=self.residual_in_fp32, eps=self.norm.eps)
        mods = self.adaLN_modulation(c).chunk(6 if self.has_text else 3, dim=1)
        x = x + mods[2].unsqueeze(1) * self.mixer(modulate(x, mods[0], mods[1]), inference_params=inference_params)
        if self.has_text:
            x = x + mods[5].unsqueeze(1) * self.msa(modulate(self.norm_msa(x), mods[3], mods[4]), text=text, mask=None)
        return x, residual


def create_block(d_model, ssm_cfg=None, has_text=False, norm_epsilon=1e-5, drop_path=0.0, rms_norm=False,
                 residual_in_fp32=False, fused_add_norm=False, skip=False, layer_idx=None, device=None,
                 dtype=None, scan_type="none", **block_kwargs):
    fk = {"device": device, "dtype": dtype}
    mixer_cls = partial(Mamba, layer_idx=layer_idx, scan_type=scan_type, **(ssm_cfg or {}), **block_kwargs, **fk)
    norm_cls = partial(nn.LayerNorm if not rms_norm else RMSNorm, eps=norm_epsilon, **fk)
    block = Block(d_model, mixer_cls, has_text=has_text, norm_cls=norm_cls, drop_path=drop_path,
                  fused_add_norm=fused_add_norm, residual_in_fp32=residual_in_fp32, skip=skip)
    block.layer_idx = layer_idx
    return block


def _init_weights(module, n_layer, initializer_range=0.02, rescale_prenorm_residual=True, n_residuals_per_layer=1):
    """model_zigma.py:512-541: zero Linear biases (unless _no_reinit), N(0, .02) embeddings, and the
    GPT-2 1/sqrt(n_layer) rescale of every out_proj / fc2 weight."""
    if isinstance(module, nn.Linear):
        if module.bias is not None and not getattr(module.bias, "_no_reinit", False):
            nn.init.zeros_(module.bias)
    elif isinstance(module, nn.Embedding):
        nn.init.normal_(module.weight, std=initializer_range)
    if rescale_prenorm_residual:
        for name, p in module.named_parameters():
            if name in ["out_proj.weight", "fc2.weight"]:
                nn.init.kaiming_uniform_(p, a=math.sqrt(5))
                with torch.no_grad():
                    p /= math.sqrt(n_residuals_per_layer * n_layer)


def get_2d_sincos_pos_embed(embed_dim, grid_size):
    """MAE-style fixed 2-D sin-cos table, (grid*grid, embed_dim), w before h (model_zigma.py:1018-1067)."""
    def one_dim(dim, pos):
        omega = 1.0 / 10000 ** (np.arange(dim // 2, dtype=np.float64) / (dim / 2.0))
        out = np.einsum("m,d->md", pos.reshape(-1), omega)
        return np.concatenate([np.sin(out), np.cos(out)], axis=1)
    gh, gw = np.arange(grid_size, dtype=np.float32), np.arange(grid_size, dtype=np.float32)
    grid = np.stack(np.meshgrid(gw, gh), axis=0).reshape(2, 1, grid_size, grid_size)
    return np.concatenate([one_dim(embed_dim // 2, grid[0]), one_dim(embed_dim // 2, grid[1])], axis=1)


class ZigMa(nn.Module):
    """A DiT-styled Mamba model with ZigZag scan."""

    def __init__(self, in_channels, embed_dim, depth, img_dim, patch_size=1, has_text=False, num_classes=-1,
                 drop_path_rate=0.1, n_context_token=0, d_context=0, ssm_cfg=None, norm_epsilon=1e-5,
                 rms_norm=True, fused_add_norm=True, residual_in_fp32=True, initializer_cfg=None,
                 scan_type="v2", video_frames=0, tpe=False, device="cuda", use_pe=0, use_jit=True,
                 m_init=True, use_checkpoint=False, dtype=torch.float32):
        self.factory_kwargs = fk = {"device": device, "dtype": dtype}
        super().__init__()
        self.in_channels = self.out_channels = in_channels
        self.patch_size, self.embed_dim, self.tpe = patch_size, embed_dim, tpe
        self.residual_in_fp32, self.fused_add_norm = residual_in_fp32, fused_add_norm
        self.video_frames, self.use_pe, self.use_checkpoint = video_frames, use_pe, use_checkpoint
        self.scan_type, self.norm_epsilon, self.img_dim = scan_type, norm_epsilon, img_dim
        num_patches = (img_dim // patch_size) ** 2
        if video_frames < 0:
            raise ValueError("video_frames should be >= 0")
        embed_cls = PatchEmbed if video_frames == 0 else PatchEmbed_Video
        self.x_embedder = embed_cls(img_dim, patch_size, in_channels, embed_dim, bias=True).to(device).to(dtype)
        self.t_embedder = TimestepEmbedder(embed_dim, dtype=dtype).to(device).to(dtype)
        n_pe = num_patches * max(video_frames, 1)
        if use_pe == 1:      # fixed sin-cos
            self.pos_embed = nn.Parameter(torch.zeros(1, n_pe, embed_dim, **fk), requires_grad=False)
        elif use_pe == 2:    # learnable
            self.pos_embed = nn.Parameter(torch.zeros(1, n_pe, embed_dim, **fk))
        elif use_pe == 3:    # per layer (a plain python list in the reference: not registered, not trained)
            self.pos_embed_list = [nn.Parameter(torch.zeros(1, n_pe, embed_dim, **fk))] * depth
        elif use_pe != 0:
            raise ValueError("use_pe should be 0, 1 or 2")
        if tpe:
            self.temporal_pos_embedding = nn.Parameter(torch.zeros(1, video_frames, embed_dim, **fk))
        self.n_layer, self.has_text, self.num_classes = depth, has_text, num_classes
        if has_text:
            self.y_embedder = nn.Linear(d_context, embed_dim).to(device).to(dtype)
        elif num_classes > 0:
            self.y_embedder = LabelEmbedder(num_classes, hidden_size=embed_dim, dropout_prob=0.0).to(device).to(dtype)
        inter_dpr = [0.0] + [x.item() for x in torch.linspace(0, drop_path_rate, depth)]
        self.drop_path = DropPath(drop_path_rate) if drop_path_rate > 0.0 else nn.Identity()

        self.extras = 0
        block_kwargs = {"use_jit": use_jit}
        block_kwargs.update(self._build_scan_tables(scan_type, depth, int(math.sqrt(num_patches)), video_frames, device))
        self.blocks = nn.ModuleList([
            create_block(embed_dim, has_text=has_text, ssm_cfg=ssm_cfg, norm_epsilon=norm_epsilon, rms_norm=rms_norm,
                         residual_in_fp32=residual_in_fp32, fused_add_norm=fused_add_norm, layer_idx=i,
                         scan_type=scan_type, drop_path=inter_dpr[i], **block_kwargs, **fk).to(device).to(dtype)
            for i in range(depth)])
        self.final_layer = FinalLayer(embed_dim, patch_size, self.out_channels).to(device).to(dtype)
        self.norm_f = (nn.LayerNorm if not rms_norm else RMSNorm)(embed_dim, eps=norm_epsilon, **fk)
        self.initialize_weights()
        self.m_init = m_init
        if m_init:
            self.apply(partial(_init_weights, n_layer=depth, **(initializer_cfg or {})))
        self._engine = None

    # ---- scan-path tables (model_zigma.py:689-794) ------------------------------------------------
    def _build_scan_tables(self, scan_type, depth, side, video_frames, device):
        to_dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(device)
        kw = {}
        if any(scan_type.startswith(p) for p in ("zigzagN", "hilbertN", "randomN", "parallelN")):
            if scan_type.startswith("zigzagN"):
                n = int(scan_type.replace("zigzagN", ""))
                paths = zigzag_path(N=side)[:n]
            elif scan_type.startswith("parallelN"):
                n = 8
                paths = zigzag_path(N=side)[:8]
            elif scan_type.startswith("hilbertN"):
                n = int(scan_type.replace("hilbertN", ""))
                paths = hilbert_path(N=side)[:n]
            else:
                n = int(scan_type.replace("randomN", ""))
                paths = []
                for _ in range(n):
                    p = np.arange(side * side)
                    np.random.shuffle(p)
                    paths.append(p)
            assert len(paths) == n, f"{len(paths)} != {n}"
            revs = [reverse_permut_np(p) for p in paths]
            kw["zigzag_paths"] = [to_dev(p) for p in paths * depth]
            kw["zigzag_paths_reverse"] = [to_dev(p) for p in revs * depth]
            kw["extras"] = self.extras
        elif scan_type.startswith("zzvideo_"):
            st_order = list(scan_type.replace("zzvideo_", ""))
            assert len(set(st_order)) == 2
            st_order = st_order * depth
            base = zigzag_path(N=side)
            zz = [to_dev(p) for p in base] * depth
            zz_rev = [to_dev(reverse_permut_np(p)) for p in base] * depth
            t_fwd = to_dev(np.arange(video_frames))
            t_bwd = to_dev(np.arange(video_frames)[::-1].copy())
            # NB the reference pairs the forward time order with the REVERSED order as its "inverse"
            # (model_zigma.py:771-772), so temporal layers hand their output back time-flipped.  Kept.
            tz, tz_rev = [t_fwd, t_bwd] * depth, [t_bwd, t_fwd] * depth
            kw["zigzag_paths"], kw["zigzag_paths_reverse"] = [], []
            for d in range(depth):
                src, src_rev = (zz, zz_rev) if st_order[d] == "s" else (tz, tz_rev)
                if st_order[d] not in "st":
                    raise ValueError("st_order should be s or t")
                kw["zigzag_paths"].append(src.pop(0))
                kw["zigzag_paths_reverse"].append(src_rev.pop(0))
            kw.update(extras=self.extras, video_frames=video_frames, st_order=st_order)
        elif scan_type != "v2":
            raise ValueError("scan_type doesn't match")
        return kw

    def initialize_weights(self):
        """model_zigma.py:840-872."""
        if self.use_pe == 1:
            pe = get_2d_sincos_pos_embed(self.pos_embed.shape[-1], int(self.x_embedder.num_patches ** 0.5))
            self.pos_embed.data.copy_(torch.from_numpy(pe).float().unsqueeze(0))
        w = self.x_embedder.proj.weight.data
        nn.init.xavier_uniform_(w.view([w.shape[0], -1]))
        nn.init.constant_(self.x_embedder.proj.bias, 0)
        nn.init.normal_(self.t_embedder.mlp[0].weight, std=0.02)
        nn.init.normal_(self.t_embedder.mlp[2].weight, std=0.02)
        for block in self.blocks:
            nn.init.constant_(block.adaLN_modulation[-1].weight, 0)
            nn.init.constant_(block.adaLN_modulation[-1].bias, 0)

    def unpatchify(self, x):
        c, p = self.out_channels, self.x_embedder.patch_size[0]
        h = w = int(x.shape[1] ** 0.5)
        assert h * w == x.shape[1]
        return x.reshape(x.shape[0], h, w, p, p, c).permute(0, 5, 1, 3, 2, 4).reshape(x.shape[0], c, h * p, w * p)

    def unpatchify_video(self, x, video_frames):
        c, p = self.out_channels, self.x_embedder.patch_size[0]
        h = w = int((x.shape[1] // video_frames) ** 0.5)
        assert h * w * video_frames == x.shape[1]
        return (x.reshape(x.shape[0], video_frames, h, w, p, p, c).permute(0, 1, 6, 2, 4, 3, 5)
                .reshape(x.shape[0], video_frames, c, h * p, w * p))

    # ---- forward ----------------------------------------------------------------------------------
    def embed(self, hidden_states, t, y=None, tokens=None, add_pos=True):
        """Everything before the blocks (model_zigma.py:923-947): tokens (B, L, D) and conditioning c.  ``tokens``: the
        patch-embedding result when the caller computed it itself (the sampling engine runs that GEMM on its wgmma kernel)."""
        hidden_states = self.x_embedder(hidden_states) if tokens is None else tokens
        _B = hidden_states.shape[0]
        t = self.t_embedder((t * 1000.0).to(hidden_states))
        if self.has_text:
            y = self.y_embedder(y)
            c = t + y.mean(dim=1)
        elif self.num_classes > 0:
            c = t + self.y_embedder(y, self.training)
        else:
            c = t
        if self.use_pe in (1, 2) and add_pos:      # (add_pos False: the sampling engine adds the table inside its first fused tail)
            hidden_states = hidden_states + self.pos_embed
        if self.video_frames > 0 and self.tpe:
            T = self.video_frames
            hs = hidden_states.reshape(_B, T, -1, hidden_states.shape[-1])
            hidden_states = (hs + self.temporal_pos_embedding.reshape(1, T, 1, -1)).reshape(hidden_states.shape)
        return hidden_states, c, y

    def forward(self, hidden_states, t, y=None):
        """x: (N, C, H, W) latents (video: (N, T, C, H, W)); t: (N,) timesteps; y: (N,) labels."""
        use_engine = (not torch.is_grad_enabled()) and (not self.training) and hidden_states.is_cuda \
            and self.fused_add_norm and self.residual_in_fp32 and self.use_pe != 3 \
            and self._engine_norms_ok()
        if use_engine:
            from .engine import ZigMaEngine
            if self._engine is None:
                self._engine = ZigMaEngine(self)
            return self._engine.forward(hidden_states, t, y)
        return self.forward_autograd(hidden_states, t, y)

    @torch.no_grad()
    def sample_euler(self, x0, num_steps=50, y=None, t0=0.0, t1=1.0, return_trajectory=False):
        """The flow-matching sampler's fixed-grid Euler loop over ``linspace(t0, t1, num_steps)`` (num_steps - 1 evaluations;
        transport/integrators.py:83-123 with sampler_type "euler") as ONE CUDA-graph replay on the sampling engine."""
        if self.training or not x0.is_cuda or not (self.fused_add_norm and self.residual_in_fp32 and self.use_pe != 3
                                                  and self._engine_norms_ok()):
            raise RuntimeError("ZigMa.sample_euler: needs an eval-mode CUDA model the sampling engine supports")
        from .engine import ZigMaEngine
        if self._engine is None:
            self._engine = ZigMaEngine(self)
        grid = torch.linspace(t0, t1, num_steps)
        return self._engine.sample_euler(x0, grid.tolist(), y, return_trajectory, dts=(grid[1:] - grid[:-1]).tolist())

    def _engine_norms_ok(self):
        """The engine's block-tail kernel is RMSNorm-only (no mean subtraction, no bias) and has no skip connection: a model
        built with rms_norm=False (nn.LayerNorm) or with skip linears samples through forward_autograd instead."""
        return (all(isinstance(b.norm, RMSNorm) and getattr(b, "skip_linear", None) is None for b in self.blocks)
                and isinstance(self.norm_f, RMSNorm))

    def _fused_tail_ok(self, hidden_states):
        """The fused training loop (block_ops.BlockTailFn) covers the configuration every shipped config uses."""
        import os
        D = hidden_states.shape[-1]
        return (hidden_states.is_cuda and self.fused_add_norm and self.residual_in_fp32 and not self.has_text and self.use_pe != 3
                and not self.use_checkpoint and D % 4 == 0 and D <= 1024 and hidden_states.dtype in (torch.float32, torch.bfloat16, torch.float16)
                and all(isinstance(b.norm, RMSNorm) and b.skip_linear is None and (isinstance(b.drop_path, nn.Identity) or not b.training)
                        for b in self.blocks)
                and isinstance(self.norm_f, RMSNorm) and (isinstance(self.drop_path, nn.Identity) or not self.training)
                and os.environ.get("ZIGMA_FUSED_TRAIN_TAIL", "1") != "0")

    def _forward_fused_tail(self, hidden_states, c):
        """Same function as the block loop of forward_autograd: each block's add+norm+modulate and the PREVIOUS block's
        gated residual add + un-permutation run as one kernel (forward and backward)."""
        from .block_ops import block_tail_fn
        from .mamba_simple import permute_along
        residual, mix, gate, rowmap = None, None, None, None
        x = hidden_states.contiguous()
        for block in self.blocks:
            mods = block.adaLN_modulation(c)
            shift, scale, gate_next = mods.chunk(3, dim=1)
            residual, x, modded = block_tail_fn(x, mix, gate, shift, scale, block.norm.weight, residual, rowmap, block.norm.eps)
            mix, rowmap = block.mixer.forward_scan_order(modded)
            gate = gate_next
        if rowmap is not None:
            mix = permute_along(mix, rowmap.long(), 1)
        return x + gate.unsqueeze(1) * mix, residual

    def forward_autograd(self, hidden_states, t, y=None):
        hidden_states, c, y = self.embed(hidden_states, t, y)
        residual = None
        if self._fused_tail_ok(hidden_states):
            hidden_states, residual = self._forward_fused_tail(hidden_states, c)
            return self._forward_head(hidden_states, residual, c)
        for layer_idx, block in enumerate(self.blocks):
            if self.use_pe == 3:
                hidden_states = hidden_states + self.pos_embed_list[layer_idx]
            if self.use_checkpoint:
                hidden_states, residual = torch.utils.checkpoint.checkpoint(
                    lambda *a: block(*a), hidden_states, residual, c, y, use_reentrant=False)
            else:
                hidden_states, residual = block(hidden_states, residual=residual, c=c, text=y)
        return self._forward_head(hidden_states, residual, c)

    def _forward_head(self, hidden_states, residual, c):
        if not self.fused_add_norm:
            residual = hidden_states if residual is None else residual + self.drop_path(hidden_states)
            hidden_states = self.norm_f(residual.to(dtype=self.norm_f.weight.dtype))
        else:
            fn = rms_norm_fn if isinstance(self.norm_f, RMSNorm) else layer_norm_fn
            hidden_states = fn(self.drop_path(hidden_states), self.norm_f.weight, self.norm_f.bias, eps=self.norm_f.eps,
                               residual=residual, prenorm=False, residual_in_fp32=self.residual_in_fp32)
        hidden_states = self.final_layer(hidden_states)
        if self.video_frames > 0:
            return self.unpatchify_video(hidden_states, self.video_frames)
        return self.unpatchify(hidden_states)

    def forward_with_cfg(self, x, t, y, cfg_scale):
        raise NotImplementedError  # as in the reference (model_zigma.py:992-993)


# model zoo (model_zigma.py:1070-1137)
def _zoo(patch_size, embed_dim, depth):
    return lambda **kwargs: ZigMa(patch_size=patch_size, embed_dim=embed_dim, depth=depth, **kwargs)


zigma_s_1, zigma_s_2, zigma_s_4 = _zoo(1, 368, 24), _zoo(2, 368, 24), _zoo(4, 368, 24)
zigma_b_1, zigma_b_2, zigma_b_4 = _zoo(1, 768, 24), _zoo(2, 768, 24), _zoo(4, 768, 24)
zigma_l_1, zigma_l_2, zigma_l_4 = _zoo(1, 1024, 48), _zoo(2, 1024, 48), _zoo(4, 1024, 48)
zigma_m_2, zigma_m_4 = _zoo(2, 768, 48), _zoo(4, 768, 48)
zigma_h_1, zigma_h_2, zigma_h_4 = _zoo(1, 1536, 48), _zoo(2, 1536, 48), _zoo(4, 1536, 48)
