"""The training step AROUND the denoiser's forward/backward kernels (SURVEY.md section 8f-1): what
``train_acc.py:436-448`` of the reference does per iteration --

    loss = transport.training_losses(model, x, model_kwargs)["loss"].mean()
    opt.zero_grad(); accelerator.backward(loss); opt.step()          # torch.optim.AdamW, DDP all-reduce inside backward
    grad_clip(opt, model, max_grad_norm); update_ema(ema_model, model)

-- laid out for an H100 node, one process per GPU:

* ``FlatParams``: every trainable parameter is a view into ONE flat fp32 buffer, every ``.grad`` a view into a
  second one (offsets 16-byte aligned).  zero_grad is one memset, the gradient norm one reduction, the
  data-parallel exchange a handful of large NCCL all-reduces over slices of one buffer, and the optimiser one
  kernel.
* ``GradSync``: bucketed all-reduce of the flat gradient buffer, launched from post-accumulate hooks as soon
  as the last gradient of a bucket exists, so the exchange over NVLink overlaps the rest of the backward
  (what DistributedDataParallel's reducer does for the reference); the 1/world mean is folded into the
  optimiser's gradient scale instead of a separate pass.
* ``FusedAdamWEMA``: AdamW + the EMA of the weights in ONE pass over the flat buffers (``zg_adamw_ema_step``,
  csrc/optim.cu) instead of AdamW's multi-pass foreach update plus two tiny launches per parameter tensor
  for the EMA (utils/train_utils.py:104-115).
"""
import copy

import torch
import torch.distributed as dist

from . import _lib

_ALIGN = 4   # elements: every parameter starts on a 16-byte boundary of the flat fp32 buffers


class FlatParams:
    """Re-homes the trainable fp32 parameters of ``module`` in one flat buffer (``.flat``) and pins their
    gradients to views of ``.grad``.  Parameter objects, names and shapes are unchanged."""

    def __init__(self, module):
        self.module = module
        self.named = [(n, p) for n, p in module.named_parameters() if p.requires_grad]
        if not self.named:
            raise ValueError("FlatParams: the module has no trainable parameters")
        dev = self.named[0][1].device
        for n, p in self.named:
            if p.dtype != torch.float32 or p.device != dev:
                raise ValueError(f"FlatParams: parameter {n} must be fp32 on {dev} (master weights; use autocast for bf16 compute)")
        self.offsets, total = [], 0
        for _, p in self.named:
            self.offsets.append(total)
            total += (p.numel() + _ALIGN - 1) // _ALIGN * _ALIGN
        self.numel = total
        self.flat = torch.zeros(total, dtype=torch.float32, device=dev)
        self.grad = torch.zeros(total, dtype=torch.float32, device=dev)
        with torch.no_grad():
            for (_, p), off in zip(self.named, self.offsets):
                v = self.flat[off:off + p.numel()].view(p.shape)
                v.copy_(p.data)
                p.data = v
                p.grad = self.grad[off:off + p.numel()].view(p.shape)
        if getattr(module, "_engine", None) is not None:
            module._engine = None          # a sampling engine built earlier packed views of the OLD parameter storage

    def view_of(self, buf, i):
        _, p = self.named[i]
        off = self.offsets[i]
        return buf[off:off + p.numel()].view(p.shape)

    def zero_grad(self):
        """One memset; the .grad views stay attached (autograd accumulates into them in place)."""
        self.grad.zero_()
        for i, (_, p) in enumerate(self.named):
            if p.grad is None or p.grad.data_ptr() != self.grad.data_ptr() + 4 * self.offsets[i]:
                p.grad = self.view_of(self.grad, i)      # somebody set it to None / replaced it

    def grad_norm(self):
        return torch.linalg.vector_norm(self.grad)


class GradSync:
    """Data-parallel mean of the flat gradient buffer, bucketed and overlapped with the backward pass."""

    def __init__(self, flat, process_group=None, bucket_mb=32.0, overlap=True):
        self.flat = flat
        self.group = process_group
        self.world = dist.get_world_size(process_group) if dist.is_available() and dist.is_initialized() else 1
        self.overlap = overlap
        if self.world > 1:
            # what DDP / accelerate do at wrap time (the reference seeds every rank differently, train_acc.py:125, and relies on
            # it): every replica starts from rank 0's weights.  The parameters are views of flat.flat, so one broadcast does it.
            dist.broadcast(flat.flat, src=dist.get_global_rank(process_group, 0) if process_group is not None else 0, group=process_group)
        # buckets = contiguous ranges of the flat buffer, filled from the END (gradients arrive in reverse order)
        cap = max(1, int(bucket_mb * (1 << 20) / 4))
        self.buckets, self.bucket_of = [], [0] * len(flat.named)
        hi = flat.numel
        members = []
        for i in range(len(flat.named) - 1, -1, -1):
            members.append(i)
            lo = flat.offsets[i]
            if hi - lo >= cap or i == 0:
                for m in members:
                    self.bucket_of[m] = len(self.buckets)
                self.buckets.append((lo, hi, len(members)))
                hi, members = lo, []
        self._pending = [0] * len(self.buckets)
        self._launched = [False] * len(self.buckets)
        self._work = []
        self._hooks = []
        if self.world > 1 and overlap:
            for i, (_, p) in enumerate(flat.named):
                self._hooks.append(p.register_post_accumulate_grad_hook(self._make_hook(i)))

    def _make_hook(self, i):
        def hook(param):
            b = self.bucket_of[i]
            self._pending[b] -= 1
            if self._pending[b] == 0:
                self._launch(b)
        return hook

    def _launch(self, b):
        if self._launched[b]:
            return
        self._launched[b] = True
        lo, hi, _ = self.buckets[b]
        self._work.append(dist.all_reduce(self.flat.grad[lo:hi], op=dist.ReduceOp.SUM, group=self.group, async_op=True))

    def begin(self):
        """Call before the backward pass of every step."""
        for b, (_, _, n) in enumerate(self.buckets):
            self._pending[b] = n
            self._launched[b] = False
        self._work = []

    def finish(self):
        """Call after backward: launches what the hooks did not (unused parameters, overlap off) and waits.
        Returns the factor that turns the summed gradients into the mean (fold it into the optimiser step)."""
        if self.world == 1:
            return 1.0
        for b in range(len(self.buckets)):
            self._launch(b)
        for w in self._work:
            w.wait()
        self._work = []
        return 1.0 / self.world

    def remove_hooks(self):
        for h in self._hooks:
            h.remove()
        self._hooks = []


class FusedAdamWEMA:
    """torch.optim.AdamW(lr, weight_decay) semantics (betas (0.9, 0.999), eps 1e-8 as the reference leaves them) plus the
    EMA of the weights, one kernel launch per step."""

    def __init__(self, flat, lr=1e-4, weight_decay=0.0, betas=(0.9, 0.999), eps=1e-8, ema_decay=0.9999, ema=True):
        if not flat.flat.is_cuda:
            raise RuntimeError("FusedAdamWEMA needs CUDA parameters (zg_adamw_ema_step has no CPU fallback)")
        self.flat = flat
        self.lr, self.weight_decay, self.betas, self.eps, self.ema_decay = lr, weight_decay, betas, eps, ema_decay
        self.exp_avg = torch.zeros_like(flat.flat)
        self.exp_avg_sq = torch.zeros_like(flat.flat)
        self.ema = flat.flat.clone() if ema else None      # update_ema(ema_model, model, decay=0) (train_acc.py:217-219)
        self.steps = 0
        self._versioned = [p for _, p in flat.named] + [flat.flat, self.exp_avg, self.exp_avg_sq] + ([self.ema] if ema else [])

    def zero_grad(self):
        self.flat.zero_grad()

    def resync_ema(self):
        """ema <- current weights (call after the weights were replaced, e.g. by GradSync's initial broadcast)."""
        if self.ema is not None:
            self.ema.copy_(self.flat.flat)

    def state_dict(self):
        """torch.optim.AdamW's layout (per-parameter 'step', 'exp_avg', 'exp_avg_sq' keyed by parameter index, one param
        group) so a reference 'opt' checkpoint entry (train_acc.py:492-501) round-trips; plus the EMA as a flat tensor."""
        state = {}
        for i, (_, p) in enumerate(self.flat.named):
            state[i] = {"step": torch.tensor(float(self.steps)), "exp_avg": self.flat.view_of(self.exp_avg, i).clone(),
                        "exp_avg_sq": self.flat.view_of(self.exp_avg_sq, i).clone()}
        group = {"lr": self.lr, "betas": tuple(self.betas), "eps": self.eps, "weight_decay": self.weight_decay, "amsgrad": False,
                 "params": list(range(len(self.flat.named)))}
        out = {"state": state, "param_groups": [group]}
        if self.ema is not None:
            out["ema_flat"] = self.ema.clone()
        return out

    def load_state_dict(self, sd):
        state, groups = sd["state"], sd["param_groups"]
        if len(state) not in (0, len(self.flat.named)):
            raise ValueError(f"FusedAdamWEMA.load_state_dict: {len(state)} parameter states for {len(self.flat.named)} parameters")
        steps = 0
        with torch.no_grad():
            for i in range(len(self.flat.named)):
                st = state.get(i, state.get(str(i)))
                if st is None:
                    continue
                self.flat.view_of(self.exp_avg, i).copy_(st["exp_avg"])
                self.flat.view_of(self.exp_avg_sq, i).copy_(st["exp_avg_sq"])
                steps = max(steps, int(float(st["step"])))
            if sd.get("ema_flat") is not None and self.ema is not None:
                self.ema.copy_(sd["ema_flat"])
        self.steps = steps
        if groups:
            g = groups[0]
            self.lr, self.betas, self.eps, self.weight_decay = g["lr"], tuple(g["betas"]), g["eps"], g["weight_decay"]

    def step(self, grad_scale=1.0, grad_scale_tensor=None):
        """grad_scale: host float (1/world, 1/loss_scale ...); grad_scale_tensor: optional fp32 device scalar multiplied
        in as well (a clip coefficient computed on the device, no host sync)."""
        self.steps += 1
        q = _lib.AdamWParams()
        q.param, q.exp_avg, q.exp_avg_sq = _lib.ptr(self.flat.flat), _lib.ptr(self.exp_avg), _lib.ptr(self.exp_avg_sq)
        q.ema, q.grad, q.grad_scale_ptr = _lib.ptr(self.ema), _lib.ptr(self.flat.grad), _lib.ptr(grad_scale_tensor)
        q.n = self.flat.numel
        q.lr, q.beta1, q.beta2, q.eps, q.weight_decay = self.lr, self.betas[0], self.betas[1], self.eps, self.weight_decay
        q.bias_correction1 = 1.0 - self.betas[0] ** self.steps
        q.bias_correction2 = 1.0 - self.betas[1] ** self.steps
        q.ema_decay, q.grad_scale = self.ema_decay, grad_scale
        _lib.call("zg_adamw_ema_step", q)
        # the kernel wrote through raw pointers: bump autograd's version counters (a parameter whose .data was pointed
        # at a view keeps its OWN counter), so that saved-tensor checks and the sampling engine's cached packed weights notice
        torch.autograd.graph.increment_version(self._versioned)

    def clip_coefficient(self, max_norm, grad_scale=1.0):
        """torch.nn.utils.clip_grad_norm_'s coefficient min(1, max_norm / (||g|| + 1e-6)) as a device scalar, and the norm."""
        norm = self.flat.grad_norm() * grad_scale
        return torch.clamp(max_norm / (norm + 1e-6), max=1.0), norm

    def ema_state_dict(self):
        """name -> EMA tensor (views of the flat EMA buffer) for the trainable parameters."""
        return {n: self.flat.view_of(self.ema, i) for i, (n, _) in enumerate(self.flat.named)}

    def ema_module(self):
        """A copy of the module whose trainable parameters ARE the EMA buffer (always current, never trained):
        the reference's ``ema_model`` (train_acc.py:210,274,285)."""
        src = self.flat.module
        eng = getattr(src, "_engine", None)      # CUDA graphs cannot be deep-copied; the copy builds its own engine on first use
        if eng is not None:
            src._engine = None
        try:
            m = copy.deepcopy(src)
        finally:
            if eng is not None:
                src._engine = eng
        byname = dict(m.named_parameters())
        for i, (n, _) in enumerate(self.flat.named):
            byname[n].data = self.flat.view_of(self.ema, i)
            byname[n].grad = None
        for p in m.parameters():
            p.requires_grad_(False)
        self._versioned += [byname[n] for n, _ in self.flat.named]      # their storage changes with every step
        return m.eval()


def train_step(model, transport, opt, sync, x1, model_kwargs=None, max_grad_norm=None, clip_before_step=False, autocast_dtype=None):
    """One iteration in the reference's order (train_acc.py:439-448).  ``max_grad_norm`` with
    ``clip_before_step=False`` reproduces the reference literally -- it clips AFTER opt.step(), i.e. the clip
    only rescales gradients that the next zero_grad discards -- so by default the norm is not even computed;
    ``clip_before_step=True`` applies the coefficient inside the fused step (no host sync).
    Returns the detached mean loss."""
    opt.zero_grad()
    if sync is not None:
        sync.begin()
    if autocast_dtype is not None:
        with torch.autocast("cuda", dtype=autocast_dtype):
            terms = transport.training_losses(model, x1, model_kwargs)
    else:
        terms = transport.training_losses(model, x1, model_kwargs)
    loss = terms["loss"].mean()
    loss.backward()
    scale = sync.finish() if sync is not None else 1.0
    coef = None
    if max_grad_norm is not None and clip_before_step:
        coef, _ = opt.clip_coefficient(max_grad_norm, scale)
    opt.step(grad_scale=scale, grad_scale_tensor=coef)
    return loss.detach()


def reference_update_ema_(ema_params, params, decay=0.9999):
    """utils/train_utils.py:104-115 restated (used by tests and the training bench as the baseline)."""
    with torch.no_grad():
        for e, p in zip(ema_params, params):
            e.mul_(decay).add_(p.data, alpha=1 - decay)


__all__ = ["FlatParams", "GradSync", "FusedAdamWEMA", "train_step", "reference_update_ema_"]
