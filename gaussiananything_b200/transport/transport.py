"""`Transport` and `Sampler` with the public surface of
/root/reference/transport/transport.py:46-489 (SiT-style flow matching).

Host-side logic only: the model evaluations it drives are the CUDA DiT kernels
when `model` is a gaussiananything_b200.dit module (any callable works).
"""
import enum
import math

import torch as th

from . import path
from .integrators import ode, sde


def mean_flat(x):
    return th.mean(x, dim=list(range(1, x.dim())))


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


class SNRType(enum.Enum):
    UNIFORM = enum.auto()
    LOGNORM = enum.auto()


class Transport:
    def __init__(self, *, model_type, path_type, loss_type, train_eps, sample_eps, snr_type):
        self.loss_type, self.model_type = loss_type, model_type
        self.path_sampler = {PathType.LINEAR: path.ICPlan, PathType.GVP: path.GVPCPlan,
                             PathType.VP: path.VPCPlan}[path_type]()
        self.train_eps, self.sample_eps, self.snr_type = train_eps, sample_eps, snr_type

    def prior_logp(self, z):
        n = z[0].numel()
        return -n / 2.0 * math.log(2 * math.pi) - th.sum(z.reshape(z.shape[0], -1) ** 2, dim=1) / 2.0

    def check_interval(self, train_eps, sample_eps, *, diffusion_form="SBDM", sde=False, reverse=False,
                       eval=False, last_step_size=0.0):
        t0, t1 = 0, 1
        eps = train_eps if not eval else sample_eps
        plan = type(self.path_sampler)
        if plan is path.VPCPlan:
            t1 = 1 - eps if (not sde or last_step_size == 0) else 1 - last_step_size
        elif plan in (path.ICPlan, path.GVPCPlan) and (self.model_type != ModelType.VELOCITY or sde):
            t0 = eps if (diffusion_form == "SBDM" and sde) or self.model_type != ModelType.VELOCITY else 0
            t1 = 1 - eps if (not sde or last_step_size == 0) else 1 - last_step_size
        if reverse:
            t0, t1 = 1 - t0, 1 - t1
        return t0, t1

    def sample(self, x1):
        """Draws (t, x0, x1) for a training pair."""
        x0 = [th.randn_like(a) for a in x1] if isinstance(x1, (list, tuple)) else th.randn_like(x1)
        t0, t1 = self.check_interval(self.train_eps, self.sample_eps)
        if self.snr_type == SNRType.UNIFORM:
            t = th.rand((len(x1),)) * (t1 - t0) + t0
        elif self.snr_type == SNRType.LOGNORM:
            t = th.sigmoid(th.normal(mean=0.0, std=1.0, size=(len(x1),))) * (t1 - t0) + t0
        else:
            raise ValueError(f"Unknown snr type: {self.snr_type}")
        return t.to(x1[0]), x0, x1

    def training_losses(self, model, x1, model_kwargs=None):
        model_kwargs = model_kwargs or {}
        t, x0, x1 = self.sample(x1)
        t, xt, ut = self.path_sampler.plan(t, x0, x1)
        out = model(xt, t, **model_kwargs)
        assert out.size() == xt.size()
        terms = {"pred": out}
        if self.model_type == ModelType.VELOCITY:
            terms["loss"] = mean_flat((out - ut) ** 2)
            return terms
        _, drift_var = self.path_sampler.compute_drift(xt, t)
        sigma_t, _ = self.path_sampler.compute_sigma_t(path.expand_t_like_x(t, xt))
        weight = {WeightType.VELOCITY: (drift_var / sigma_t) ** 2, WeightType.LIKELIHOOD: drift_var / (sigma_t ** 2),
                  WeightType.NONE: 1}[self.loss_type]
        target = (out - x0) if self.model_type == ModelType.NOISE else (out * sigma_t + x0)
        terms["loss"] = mean_flat(weight * target ** 2)
        return terms

    def get_drift(self):
        """Drift of the probability-flow ODE for the model's parametrisation."""
        ps = self.path_sampler

        def score_ode(x, t, model, **kw):
            mean, var = ps.compute_drift(x, t)
            return -mean + var * model(x, t, **kw)

        def noise_ode(x, t, model, **kw):
            mean, var = ps.compute_drift(x, t)
            sigma_t, _ = ps.compute_sigma_t(path.expand_t_like_x(t, x))
            return -mean + var * (model(x, t, **kw) / -sigma_t)

        def velocity_ode(x, t, model, **kw):
            return model(x, t, **kw)

        fn = {ModelType.NOISE: noise_ode, ModelType.SCORE: score_ode, ModelType.VELOCITY: velocity_ode}[self.model_type]

        def body_fn(x, t, model, **kw):
            out = fn(x, t, model, **kw)
            assert out.shape == x.shape, "Output shape from ODE solver must match input shape"
            return out

        return body_fn

    def get_score(self):
        ps = self.path_sampler
        if self.model_type == ModelType.NOISE:
            return lambda x, t, model, **kw: model(x, t, **kw) / -ps.compute_sigma_t(path.expand_t_like_x(t, x))[0]
        if self.model_type == ModelType.SCORE:
            return lambda x, t, model, **kw: model(x, t, **kw)
        if self.model_type == ModelType.VELOCITY:
            return lambda x, t, model, **kw: ps.get_score_from_velocity(model(x, t, **kw), x, t)
        raise NotImplementedError()


class Sampler:
    """Sampler(transport).sample_ode(...) -> fn(x, model, **model_kwargs) -> trajectory [num_steps, *x.shape]."""

    def __init__(self, transport, guider_config=None):
        self.transport = transport
        self.drift = transport.get_drift()
        self.score = transport.get_score()

    def sample_ode(self, *, sampling_method="dopri5", num_steps=50, atol=1e-6, rtol=1e-3, reverse=False, cfg=False):
        drift = self.drift
        if reverse:
            drift = lambda x, t, model, **kw: self.drift(x, th.ones_like(t) * (1 - t), model, **kw)
        t0, t1 = self.transport.check_interval(self.transport.train_eps, self.transport.sample_eps, sde=False,
                                               eval=True, reverse=reverse, last_step_size=0.0)
        return ode(drift=drift, t0=t0, t1=t1, sampler_type=sampling_method, num_steps=num_steps, atol=atol,
                   rtol=rtol).sample

    def sample_sde(self, *, sampling_method="Euler", diffusion_form="SBDM", diffusion_norm=1.0, last_step="Mean",
                   last_step_size=0.04, num_steps=250):
        if last_step is None:
            last_step_size = 0.0
        ps = self.transport.path_sampler
        diffusion_fn = lambda x, t: ps.compute_diffusion(x, t, form=diffusion_form, norm=diffusion_norm)
        sde_drift = lambda x, t, model, **kw: self.drift(x, t, model, **kw) + diffusion_fn(x, t) * self.score(x, t, model, **kw)
        t0, t1 = self.transport.check_interval(self.transport.train_eps, self.transport.sample_eps,
                                               diffusion_form=diffusion_form, sde=True, eval=True, reverse=False,
                                               last_step_size=last_step_size)
        _sde = sde(sde_drift, diffusion_fn, t0=t0, t1=t1, num_steps=num_steps, sampler_type=sampling_method)
        if last_step is None:
            last_fn = lambda x, t, model, **kw: x
        elif last_step == "Mean":
            last_fn = lambda x, t, model, **kw: x + sde_drift(x, t, model, **kw) * last_step_size
        elif last_step == "Tweedie":
            last_fn = lambda x, t, model, **kw: x / ps.compute_alpha_t(t)[0][0] + \
                (ps.compute_sigma_t(t)[0][0] ** 2) / ps.compute_alpha_t(t)[0][0] * self.score(x, t, model, **kw)
        elif last_step == "Euler":
            last_fn = lambda x, t, model, **kw: x + self.drift(x, t, model, **kw) * last_step_size
        else:
            raise NotImplementedError()

        def _sample(init, model, **kw):
            xs = _sde.sample(init, model, **kw)
            ts = th.ones(init.size(0), device=init.device) * t1
            xs.append(last_fn(xs[-1], ts, model, **kw))
            assert len(xs) == num_steps, "Samples does not match the number of steps"
            return xs

        return _sample

    def sample_ode_likelihood(self, *, sampling_method="dopri5", num_steps=50, atol=1e-6, rtol=1e-3):
        """Hutchinson-trace likelihood ODE (reference transport.py:433-489); fixed-grid or dopri5 on the
        concatenated (x, logp) state."""
        drift_fn = self.drift
        t0, t1 = self.transport.check_interval(self.transport.train_eps, self.transport.sample_eps, sde=False,
                                               eval=True, reverse=False, last_step_size=0.0)
        from .integrators import odeint

        def _sample_fn(x, model, **kw):
            shape, n = x.shape, x[0].numel()

            def f(t, state):
                xx = state[:, :n].reshape(shape)
                tb = th.ones(xx.size(0), device=xx.device) * (1 - t)
                eps = th.randint(2, xx.size(), dtype=th.float, device=xx.device) * 2 - 1
                with th.enable_grad():
                    xx = xx.detach().requires_grad_(True)
                    d = drift_fn(xx, tb, model, **kw)
                    grad = th.autograd.grad(th.sum(d * eps), xx)[0]
                logp_grad = th.sum(grad * eps, dim=tuple(range(1, xx.dim())))
                return th.cat([(-d.detach()).reshape(xx.size(0), n), logp_grad[:, None]], 1)

            state0 = th.cat([x.reshape(x.size(0), n), th.zeros(x.size(0), 1).to(x)], 1)
            ts = th.linspace(t0, t1, num_steps).to(x.device)
            out = odeint(f, state0, ts, method=sampling_method, atol=atol, rtol=rtol)[-1]
            z, delta = out[:, :n].reshape(shape), out[:, n]
            return self.transport.prior_logp(z) - delta, z

        return _sample_fn
