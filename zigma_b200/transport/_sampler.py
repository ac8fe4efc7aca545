"""Transport / Sampler / sde / ode of the reference's ``transport/transport.py`` and
``transport/integrators.py`` -- the host-side loop that DRIVES the denoiser hot path (one or more
``model(x, t, **kw)`` evaluations per step; each is one ZigMaEngine graph replay on the GPU).

Random draws follow the reference exactly (what is drawn, in which order, from which generator:
CPU ``torch.randn(x.size()).to(x)`` in the SDE steps, integrators.py:33,43; CPU ``torch.rand`` for
the training time, transport.py:122), so a seeded run reproduces the reference's stream.
"""
import enum
import math

import torch

from . import _plans as path
from ._odeint import odeint


def mean_flat(x):
    """Mean over all non-batch dims (transport/utils.py:13-17)."""
    return torch.mean(x, dim=list(range(1, x.dim())))


class EasyDict:
    """transport/utils.py:3-11."""

    def __init__(self, sub_dict):
        for k, v in sub_dict.items():
            setattr(self, k, v)

    def __getitem__(self, key):
        return getattr(self, key)


class ModelType(enum.Enum):
    NOISE = enum.auto()
    SCORE = enum.auto()
    VELOCITY = enum.auto()


class PathType(enum.Enum):
    LINEAR = enum.auto()
    GVP = enum.auto()
    VP = enum.auto()


class WeightType(enum.Enum):
    NONE = enum.auto()
    VELOCITY = enum.auto()
    LIKELIHOOD = enum.auto()


_PLANS = {PathType.LINEAR: path.ICPlan, PathType.GVP: path.GVPCPlan, PathType.VP: path.VPCPlan}


class Transport:
    """transport/transport.py:43-233."""

    def __init__(self, *, model_type, path_type, loss_type, train_eps, sample_eps):
        self.loss_type, self.model_type = loss_type, model_type
        self.path_type = path_type
        self.path_sampler = _PLANS[path_type]()
        self.train_eps, self.sample_eps = train_eps, sample_eps

    def prior_logp(self, z):
        """Standard-normal log density per batch element (transport.py:68-76)."""
        n = z[0].numel()
        return -n / 2.0 * math.log(2 * math.pi) - z.flatten(1).pow(2).sum(1) / 2.0

    def check_interval(self, train_eps, sample_eps, *, diffusion_form="SBDM", sde=False, reverse=False,
                       eval=False, last_step_size=0.0):
        """Integration interval with the singular ends trimmed (transport.py:78-112)."""
        t0, t1 = 0, 1
        eps = sample_eps if eval else train_eps
        is_vp = type(self.path_sampler) is path.VPCPlan
        velocity = self.model_type == ModelType.VELOCITY
        if is_vp or (not velocity or sde):
            if not is_vp:
                t0 = eps if ((diffusion_form == "SBDM" and sde) or not velocity) else 0
            t1 = 1 - eps if (not sde or last_step_size == 0) else 1 - last_step_size
        if reverse:
            t0, t1 = 1 - t0, 1 - t1
        return t0, t1

    def sample(self, x1):
        """Draw (t, x0) for a data batch x1 (transport.py:114-124)."""
        x0 = torch.randn_like(x1)
        t0, t1 = self.check_interval(self.train_eps, self.sample_eps)
        t = (torch.rand((x1.shape[0],)) * (t1 - t0) + t0).to(x1)
        return t, x0, x1

    def training_losses(self, model, x1, model_kwargs=None):
        """Flow-matching / score-matching loss (transport.py:126-173): returns {"pred", "loss"} with a
        per-sample loss."""
        model_kwargs = {} if model_kwargs is None else model_kwargs
        t, x0, x1 = self.sample(x1)
        t, xt, ut = self.path_sampler.plan(t, x0, x1)
        out = model(xt, t, **model_kwargs)
        assert out.size() == xt.size(), f"Model output shape {out.size()} does not match input shape {xt.size()}"
        terms = {"pred": out}
        if self.model_type == ModelType.VELOCITY:
            terms["loss"] = mean_flat((out - ut) ** 2)
            return terms
        _, drift_var = self.path_sampler.compute_drift(xt, t)
        sigma_t, _ = self.path_sampler.compute_sigma_t(path.expand_t_like_x(t, xt))
        if self.loss_type == WeightType.VELOCITY:
            weight = (drift_var / sigma_t) ** 2
        elif self.loss_type == WeightType.LIKELIHOOD:
            weight = drift_var / (sigma_t ** 2)
        elif self.loss_type == WeightType.NONE:
            weight = 1
        else:
            raise NotImplementedError()
        if self.model_type == ModelType.NOISE:
            terms["loss"] = mean_flat(weight * ((out - x0) ** 2))
        elif self.model_type == ModelType.SCORE:
            terms["loss"] = mean_flat(weight * ((out * sigma_t + x0) ** 2))
        else:
            raise NotImplementedError()
        return terms

    def get_drift(self):
        """Probability-flow ODE drift for the model's parametrisation (transport.py:175-210)."""
        plan, mtype = self.path_sampler, self.model_type
        if mtype not in (ModelType.NOISE, ModelType.SCORE, ModelType.VELOCITY):
            raise NotImplementedError()

        def body_fn(x, t, model, **model_kwargs):
            if mtype == ModelType.VELOCITY:
                out = model(x, t, **model_kwargs)
            else:
                drift_mean, drift_var = plan.compute_drift(x, t)
                if mtype == ModelType.NOISE:
                    sigma_t, _ = plan.compute_sigma_t(path.expand_t_like_x(t, x))
                    score = model(x, t, **model_kwargs) / -sigma_t
                else:
                    score = model(x, t, **model_kwargs)
                out = -drift_mean + drift_var * score
            assert out.shape == x.shape, "Output shape from ODE solver must match input shape"
            return out

        return body_fn

    def get_score(self):
        """Score of p_t from the model output (transport.py:212-233)."""
        plan, mtype = self.path_sampler, self.model_type
        if mtype == ModelType.NOISE:
            return lambda x, t, model, **kw: model(x, t, **kw) / -plan.compute_sigma_t(path.expand_t_like_x(t, x))[0]
        if mtype == ModelType.SCORE:
            return lambda x, t, model, **kw: model(x, t, **kw)
        if mtype == ModelType.VELOCITY:
            return lambda x, t, model, **kw: plan.get_score_from_velocity(model(x, t, **kw), x, t)
        raise NotImplementedError()


class sde:
    """Fixed-step SDE integrator (transport/integrators.py:9-80): Euler-Maruyama or stochastic Heun
    over ``linspace(t0, t1, num_steps)``; ``sample`` returns the num_steps-1 intermediate states."""

    def __init__(self, drift, diffusion, *, t0, t1, num_steps, sampler_type):
        assert t0 < t1, "SDE sampler has to be in forward time"
        self.num_timesteps = num_steps
        self.t = torch.linspace(t0, t1, num_steps)
        self.dt = self.t[1] - self.t[0]
        self.drift, self.diffusion, self.sampler_type = drift, diffusion, sampler_type

    def _noise(self, x):
        return torch.randn(x.size()).to(x) * torch.sqrt(self.dt)

    @staticmethod
    def _amp(diffusion):
        # the reference's torch.sqrt(2 * diffusion) raises for the python-float "constant" form
        # (integrators.py:39); accept it.
        return torch.sqrt(2 * diffusion) if torch.is_tensor(diffusion) else math.sqrt(2 * diffusion)

    def _euler_maruyama(self, x, t, model, **kw):
        dw = self._noise(x)
        tb = torch.ones(x.size(0)).to(x) * t
        mean_x = x + self.drift(x, tb, model, **kw) * self.dt
        return mean_x + self._amp(self.diffusion(x, tb)) * dw

    def _heun(self, x, t, model, **kw):
        dw = self._noise(x)
        tb = torch.ones(x.size(0)).to(x) * t
        xhat = x + self._amp(self.diffusion(x, tb)) * dw
        k1 = self.drift(xhat, tb, model, **kw)
        k2 = self.drift(xhat + self.dt * k1, tb + self.dt, model, **kw)
        return xhat + 0.5 * self.dt * (k1 + k2)

    def sample(self, init, model, **model_kwargs):
        try:
            step = {"Euler": self._euler_maruyama, "Heun": self._heun}[self.sampler_type]
        except KeyError:
            raise NotImplementedError("Smapler type not implemented.")
        x, samples = init, []
        with torch.no_grad():
            for ti in self.t[:-1]:
                x = step(x, ti, model, **model_kwargs)
                samples.append(x)
        return samples


class ode:
    """ODE driver (transport/integrators.py:83-123): hands ``linspace(t0, t1, num_steps)`` to odeint
    (here zigma_b200.transport._odeint, the restated torchdiffeq) with per-tensor tolerances."""

    def __init__(self, drift, *, t0, t1, sampler_type, num_steps, atol, rtol):
        self.drift = drift
        self.t = torch.linspace(t0, t1, num_steps)
        self.atol, self.rtol, self.sampler_type = atol, rtol, sampler_type

    def sample(self, x, model, **model_kwargs):
        multi = isinstance(x, tuple)
        lead = x[0] if multi else x
        device = lead.device

        def fn(t, state):
            n = state[0].size(0) if isinstance(state, tuple) else state.size(0)
            return self.drift(state, torch.ones(n).to(device) * t, model, **model_kwargs)

        k = len(x) if multi else 1
        return odeint(fn, x, self.t.to(device), method=self.sampler_type, atol=[self.atol] * k, rtol=[self.rtol] * k)


class Sampler:
    """transport/transport.py:236-476: builds the sampling closures."""

    def __init__(self, transport):
        self.transport = transport
        self.drift = transport.get_drift()
        self.score = transport.get_score()

    def _sde_terms(self, diffusion_form, diffusion_norm):
        plan = self.transport.path_sampler
        diffusion = lambda x, t: plan.compute_diffusion(x, t, form=diffusion_form, norm=diffusion_norm)
        drift = lambda x, t, model, **kw: self.drift(x, t, model, **kw) + diffusion(x, t) * self.score(x, t, model, **kw)
        return drift, diffusion

    def _last_step(self, sde_drift, last_step, last_step_size):
        """transport.py:272-308."""
        if last_step is None:
            return lambda x, t, model, **kw: x
        if last_step == "Mean":
            return lambda x, t, model, **kw: x + sde_drift(x, t, model, **kw) * last_step_size
        if last_step == "Tweedie":
            alpha, sigma = self.transport.path_sampler.compute_alpha_t, self.transport.path_sampler.compute_sigma_t
            return lambda x, t, model, **kw: (x / alpha(t)[0][0]
                                              + (sigma(t)[0][0] ** 2) / alpha(t)[0][0] * self.score(x, t, model, **kw))
        if last_step == "Euler":
            return lambda x, t, model, **kw: x + self.drift(x, t, model, **kw) * last_step_size
        raise NotImplementedError()

    def sample_sde(self, *, sampling_method="Euler", diffusion_form="SBDM", diffusion_norm=1.0, last_step="Mean",
                   last_step_size=0.04, num_steps=250):
        """transport.py:310-370: returns ``fn(init_z, model, **kw) -> list of num_steps states``."""
        if last_step is None:
            last_step_size = 0.0
        sde_drift, sde_diffusion = self._sde_terms(diffusion_form, diffusion_norm)
        tr = self.transport
        t0, t1 = tr.check_interval(tr.train_eps, tr.sample_eps, diffusion_form=diffusion_form, sde=True, eval=True,
                                   reverse=False, last_step_size=last_step_size)
        solver = sde(sde_drift, sde_diffusion, t0=t0, t1=t1, num_steps=num_steps, sampler_type=sampling_method)
        last = self._last_step(sde_drift, last_step, last_step_size)

        def _sample(init_z, model, **model_kwargs):
            xs = solver.sample(init_z, model, **model_kwargs)
            ts = torch.ones(init_z.size(0), device=init_z.device) * t1
            xs.append(last(xs[-1], ts, model, **model_kwargs))
            assert len(xs) == num_steps, "Samples does not match the number of steps"
            return xs

        return _sample

    def sample_ode(self, *, sampling_method="dopri5", num_steps=50, atol=1e-6, rtol=1e-3, reverse=False):
        """transport.py:372-417: returns ``fn(x, model, **kw) -> (num_steps, ...) trajectory``."""
        if reverse:
            drift = lambda x, t, model, **kw: self.drift(x, torch.ones_like(t) * (1 - t), model, **kw)
        else:
            drift = self.drift
        tr = self.transport
        t0, t1 = tr.check_interval(tr.train_eps, tr.sample_eps, sde=False, eval=True, reverse=reverse, last_step_size=0.0)
        return ode(drift=drift, t0=t0, t1=t1, sampler_type=sampling_method, num_steps=num_steps, atol=atol, rtol=rtol).sample

    def sample_ode_likelihood(self, *, sampling_method="dopri5", num_steps=50, atol=1e-6, rtol=1e-3):
        """transport.py:418-476: integrates data -> noise with a Hutchinson (Rademacher) trace estimate
        of the divergence; returns ``fn(x, model, **kw) -> (logp, z)``."""

        def likelihood_drift(state, t, model, **kw):
            x, _ = state
            eps = torch.randint(2, x.size(), dtype=torch.float, device=x.device) * 2 - 1
            t = torch.ones_like(t) * (1 - t)
            with torch.enable_grad():
                x = x.detach().requires_grad_(True)     # (the reference flips the flag in place, transport.py:442)
                grad = torch.autograd.grad(torch.sum(self.drift(x, t, model, **kw) * eps), x)[0]
                logp_grad = torch.sum(grad * eps, dim=tuple(range(1, x.dim())))
                drift = self.drift(x, t, model, **kw)
            return -drift.detach(), logp_grad.detach()      # keep the solver state graph-free

        tr = self.transport
        t0, t1 = tr.check_interval(tr.train_eps, tr.sample_eps, sde=False, eval=True, reverse=False, last_step_size=0.0)
        solver = ode(drift=likelihood_drift, t0=t0, t1=t1, sampler_type=sampling_method, num_steps=num_steps,
                     atol=atol, rtol=rtol)

        def _sample_fn(x, model, **model_kwargs):
            z, delta_logp = solver.sample((x, torch.zeros(x.size(0)).to(x)), model, **model_kwargs)
            z, delta_logp = z[-1], delta_logp[-1]
            return self.transport.prior_logp(z) - delta_logp, z

        return _sample_fn
