"""Flow-matching sampler with the reference's ``transport`` API for the path VisualCloze uses.

  create_transport  transport/__init__.py:4-62       Sampler.sample_ode  transport/transport.py:361-410
  ode grid          transport/integrators.py:79-120  time_shift          transport/utils.py:33-43
  velocity_ode      transport/transport.py:193-198   fixed-grid solvers  torchdiffeq.odeint(method="euler" | "midpoint" | "rk4")

``Sampler(transport).sample_ode(...)`` returns ``fn(x, model, model_kwargs)`` which returns the whole trajectory
``[num_steps, B, L, C]`` (callers index ``[-1]``).  ``num_steps`` time points mean ``num_steps - 1`` model
evaluations.  When ``model`` is the bound ``forward`` of a ``visualcloze_b200.model.Flux`` the step-invariant work
of all evaluations, stage evaluations included, is hoisted (one engine.prepare) and each evaluation is one
``vcb_flux_forward`` followed by one ``vcb_ode_stage``; any other callable is driven evaluation by evaluation through the same
stage kernel.

Only what the inference pipeline uses is implemented: Linear path, velocity prediction and torchdiffeq's fixed-grid solvers
"euler", "midpoint" and "rk4" (DESIGN.md 2e).  Training losses, SDE samplers, likelihood ODE, VP/GVP paths and adaptive
solvers are out of scope (SURVEY.md 2 #6).
"""
from __future__ import annotations

import enum
import math

import torch as th

from . import ops


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


def time_shift(mu: float, sigma: float, t: th.Tensor):
    """transport/utils.py:33-38: the mirrored (t=0 noise, t=1 data) form of the FLUX shift."""
    t = 1 - t
    t = math.exp(mu) / (math.exp(mu) + (1 / t - 1) ** sigma)
    t = 1 - t
    return t


def get_lin_function(x1: float = 256, y1: float = 0.5, x2: float = 4096, y2: float = 1.15):
    m = (y2 - y1) / (x2 - x1)
    b = y1 - m * x1
    return lambda x: m * x + b


class Transport:
    def __init__(self, *, model_type, path_type, loss_type="mse", train_eps=0, sample_eps=0, snr_type="uniform",
                 do_shift=True):
        if path_type != PathType.LINEAR or model_type != ModelType.VELOCITY:
            raise NotImplementedError("only the Linear path with velocity prediction is on the VisualCloze inference path")
        self.model_type, self.path_type = model_type, path_type
        self.loss_type, self.train_eps, self.sample_eps = loss_type, train_eps, sample_eps
        self.snr_type, self.do_shift = snr_type, do_shift

    def check_interval(self, train_eps, sample_eps, *, diffusion_form="SBDM", sde=False, reverse=False, eval=False,
                       last_step_size=0.0):
        t0, t1 = 0, 1          # Linear + velocity "is stable everywhere" (transport/transport.py:70-96)
        if reverse:
            t0, t1 = 1 - t0, 1 - t1
        return t0, t1


def create_transport(path_type="Linear", prediction="velocity", loss_weight=None, train_eps=None, sample_eps=None,
                     snr_type="uniform", loss_type="mse", do_shift=True):
    model_type = {"noise": ModelType.NOISE, "score": ModelType.SCORE}.get(prediction, ModelType.VELOCITY)
    ptype = {"Linear": PathType.LINEAR, "GVP": PathType.GVP, "VP": PathType.VP}[path_type]
    return Transport(model_type=model_type, path_type=ptype, loss_type=loss_type, train_eps=0, sample_eps=0,
                     snr_type=snr_type, do_shift=do_shift)


def solver_grid(t0, t1, num_steps: int, seq_len: int, do_shift: bool, time_shifting_factor) -> th.Tensor:
    """integrators.py:99-101 and :114-116 -- fp32 grid of solver time (0 = noise, 1 = data)."""
    t = th.linspace(t0, t1, int(num_steps))
    if time_shifting_factor:
        t = t / (t + time_shifting_factor - time_shifting_factor * t)
    if do_shift:
        mu = get_lin_function(y1=0.5, y2=1.15)(seq_len)
        t = time_shift(mu, 1.0, t)
    return t


def _is_native_forward(model) -> bool:
    from .model import Flux
    return isinstance(getattr(model, "__self__", None), Flux) and getattr(model, "__name__", "") == "forward"


_ONE_THIRD = 1 / 3                   # torchdiffeq/_impl/rk_common.py: _one_third, _two_thirds (Python floats)
_TWO_THIRDS = 2 / 3
SUPPORTED_METHODS = tuple(ops.ODE_STAGES)      # ("euler", "midpoint", "rk4")


def stage_times(t: th.Tensor, method: str) -> th.Tensor:
    """[N - 1, stages] fp32 solver times of every model evaluation on the grid ``t``, in evaluation order, formed by the fp32
    tensor ops torchdiffeq applies per interval (t0, t1 0-dim fp32, dt = t1 - t0):
      euler     t0
      midpoint  t0, t0 + half_dt                        half_dt = 0.5 * dt              (fixed_grid.py Midpoint)
      rk4       t0, t0 + dt * _one_third, t0 + dt * _two_thirds, t1                     (rk_common.py rk4_alt_step_func)"""
    t0, t1 = t[:-1], t[1:]
    dt = t1 - t0
    cols = {"euler": lambda: [t0],
            "midpoint": lambda: [t0, t0 + 0.5 * dt],
            "rk4": lambda: [t0, t0 + dt * _ONE_THIRD, t0 + dt * _TWO_THIRDS, t1]}[method]()
    return th.stack(cols, dim=1)


class Sampler:
    """Sampler class for the transport model (fixed-grid ODE solvers: euler, midpoint, rk4)."""

    def __init__(self, transport: Transport):
        self.transport = transport

    def sample_ode(self, *, sampling_method="dopri5", num_steps=50, atol=1e-6, rtol=1e-3, reverse=False, do_shift=True,
                   time_shifting_factor=None, strength=None):
        if sampling_method not in SUPPORTED_METHODS:
            raise NotImplementedError(f"sampling_method={sampling_method!r}: only the fixed-grid solvers "
                                      f"{', '.join(map(repr, SUPPORTED_METHODS))} are implemented (adaptive solvers are not)")
        t0, t1 = self.transport.check_interval(self.transport.train_eps, self.transport.sample_eps, sde=False, eval=True,
                                               reverse=reverse, last_step_size=0.0)
        if strength is not None:
            t0 = (t1 - t0) * strength + t0
        assert t0 < t1, "ODE sampler has to be in forward time"

        def _sample(x, model, model_kwargs):
            return _fixed_grid_sample(x, model, model_kwargs, sampling_method, t0, t1, num_steps, do_shift, time_shifting_factor)

        return _sample


def _fixed_grid_sample(x, model, model_kwargs, method, t0, t1, num_steps, do_shift, time_shifting_factor):
    if not (x.is_cuda and x.dtype == th.bfloat16):
        raise ops._lib.VcbError("the sampler runs on CUDA bf16 latents only (visualcloze.py:399); there is no CPU path")
    B, Li, C = x.shape
    t = solver_grid(t0, t1, num_steps, Li, do_shift, time_shifting_factor)
    n_int = int(num_steps) - 1
    stages = ops.ODE_STAGES[method]
    n_eval = stages * n_int                       # evaluation e = k * stages + s: stage s of interval k
    kw = dict(model_kwargs)                       # the caller's dict is not mutated (transport.py:194-196 pops a copy)
    cond = kw.pop("cond", None)
    # FLUX time fed to the model: ones(B) * t -> 1 - t (integrators.py:109, transport.py:384), fp32.  torchdiffeq wraps the
    # ODE function in _PerturbFunc, which casts the evaluation time to the STATE dtype (t.to(y.abs().dtype)): with the bf16
    # latent the model sees 1 - bf16(tau) (up to ~2 units of 1000 t near tau = 1).  The stage times are fp32 ops on the grid.
    t_vec = th.ones(n_eval, B) * stage_times(t, method).reshape(n_eval, 1).to(x.dtype).float()
    flux_t = th.ones_like(t_vec) * (1 - t_vec)
    # dt is the fp32 t1 - t0; the stage kernel applies it as torch does a 0-dim fp32 tensor in a bf16 op (vcb_ode_stage)
    dts = [float(t[k + 1] - t[k]) for k in range(n_int)]

    native = _is_native_forward(model)
    sp = model.__self__.engine()._sp if native else None
    if sp is not None:
        # single-image sequence parallelism: this rank integrates its own token rows (every stage update is row-local; only
        # the attention inside the model mixes rows); the trajectory is gathered once at the end.  The grid used the FULL Li.
        x = sp.shard(x).contiguous()
        cond = None if cond is None else sp.shard(cond)
    Li_full, Li = Li, x.shape[1]
    traj = th.empty(int(num_steps), B, Li, C, dtype=x.dtype, device=x.device)
    traj[0].copy_(x)
    Cc = 0 if cond is None else cond.shape[-1]
    inp = th.empty(B, Li, C + Cc, dtype=x.dtype, device=x.device)       # cat(x, cond) buffer (transport.py:195)
    ops.copy_cols(traj[0].reshape(B * Li, C), inp.reshape(B * Li, C + Cc), 0)
    if cond is not None:
        ops.copy_cols(cond.to(x.dtype).reshape(B * Li, Cc).contiguous(), inp.reshape(B * Li, C + Cc), C)
    y_stage = th.empty(B * Li, C, dtype=x.dtype, device=x.device) if stages > 1 else None   # stage states are not returned

    if native:
        flux = model.__self__
        eng = flux.engine()
        if flux.params.guidance_embed and kw.get("guidance") is None:
            raise ValueError("Didn't get guidance strength for guidance distilled model.")
        eng.prepare(txt=kw["txt"], y=kw["y"], img_ids=kw["img_ids"], txt_ids=kw["txt_ids"], timesteps=flux_t,
                    guidance=kw.get("guidance"), txt_mask=kw.get("txt_mask"), img_mask=kw.get("img_mask"), n_img_tokens=Li_full)
        v = th.empty(stages, B, Li, flux.params.out_channels, dtype=x.dtype, device=x.device)
    for k in range(n_int):
        vs = []
        for s in range(stages):
            e = k * stages + s
            if native:
                out = eng.forward(e, inp, v[s])
            else:
                out = model(inp, timesteps=flux_t[e].to(x.device), **kw)
            assert out.shape == x.shape, "Output shape from ODE solver must match input shape"
            vs.append(out.reshape(B * Li, C))
            y_out = traj[k + 1].reshape(B * Li, C) if s == stages - 1 else y_stage
            ops.ode_stage(method, s, traj[k].reshape(B * Li, C), vs, dts[k], y_out, inp.reshape(B * Li, C + Cc))
    if sp is not None:
        traj = sp.gather(traj, dim=2)
        sp.check()
    return traj
