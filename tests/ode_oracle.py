"""Restatement of torchdiffeq's fixed-grid "midpoint" and "rk4" solvers for the tests -- TEST INFRASTRUCTURE ONLY.

``oracle/sampler_oracle.py`` restates the reference sampler with the fixed-grid Euler solver, and the torchdiffeq stand-in that
``oracle/build_ref.py`` writes into ``oracle/_ref`` implements Euler only.  This module extends both to the two other classic
fixed-grid solvers of torchdiffeq (torchdiffeq/_impl/fixed_grid.py, rk_common.py; unpinned, not vendored by the reference), one
interval [t0, t1] at a time, ``dt = t1 - t0`` a 0-dim fp32 tensor, every line one eager torch op on the state:

  euler     y1 = y0 + dt * f(t0, y0)
  midpoint  half_dt = 0.5 * dt; k1 = f(t0, y0); k2 = f(t0 + half_dt, y0 + k1 * half_dt); y1 = y0 + dt * k2
  rk4       rk4_alt_step_func, the 3/8 rule: k1 = f(t0, y0), k2 = f(t0 + dt * _one_third, y0 + dt * k1 * _one_third),
            k3 = f(t0 + dt * _two_thirds, y0 + dt * (k2 - k1 * _one_third)), k4 = f(t1, y0 + dt * (k1 - k2 + k3)),
            y1 = y0 + (k1 + 3 * (k2 + k3) + k4) * dt * 0.125

  * ``sample_ode(..., method=)`` is ``sampler_oracle.sample_ode`` with these solvers (its Euler equals that oracle bit for bit);
  * ``odeint`` is a drop-in for the stand-in's ``odeint`` with the same structure as upstream (``_PerturbFunc``'s cast of the
    time to the state dtype, ``y1 = y0 + dy``); a test installs it as ``transport.integrators.odeint`` of the UNMODIFIED
    reference package, so the reference's own sampler drives these solvers.
"""
from __future__ import annotations

import torch

from oracle import sampler_oracle

_one_third = 1 / 3
_two_thirds = 2 / 3
METHODS = ("euler", "midpoint", "rk4")


def _euler(func, t0, dt, t1, y0):
    return dt * func(t0, y0)


def _midpoint(func, t0, dt, t1, y0):
    half_dt = 0.5 * dt
    f0 = func(t0, y0)
    y_mid = y0 + f0 * half_dt
    return dt * func(t0 + half_dt, y_mid)


def _rk4(func, t0, dt, t1, y0):
    k1 = func(t0, y0)
    k2 = func(t0 + dt * _one_third, y0 + dt * k1 * _one_third)
    k3 = func(t0 + dt * _two_thirds, y0 + dt * (k2 - k1 * _one_third))
    k4 = func(t1, y0 + dt * (k1 - k2 + k3))
    return (k1 + 3 * (k2 + k3) + k4) * dt * 0.125


_STEPS = {"euler": _euler, "midpoint": _midpoint, "rk4": _rk4}


def odeint(func, y0, t, *, rtol=1e-7, atol=1e-9, method=None, options=None, event_fn=None):
    """torchdiffeq.odeint for the fixed-grid euler / midpoint / rk4 solvers: the stacked trajectory at the grid points."""
    if method not in _STEPS:
        raise NotImplementedError(f"fixed-grid {METHODS} only, not {method!r}")
    t = t.to(y0.device)
    step = _STEPS[method]

    def perturbed(tt, y):                       # _PerturbFunc.forward: t.to(y.abs().dtype)
        return func(tt.to(y.abs().dtype), y)

    solution = torch.empty(len(t), *y0.shape, dtype=y0.dtype, device=y0.device)
    solution[0] = y0
    y = y0
    for j in range(1, len(t)):
        t0, t1 = t[j - 1], t[j]
        y = y + step(perturbed, t0, t1 - t0, t1, y)
        solution[j] = y
    return solution


def sample_ode(x: torch.Tensor, model_fn, model_kwargs: dict, num_steps: int, do_shift: bool = True, time_shifting_factor=None,
               strength=None, method: str = "euler") -> torch.Tensor:
    """``sampler_oracle.sample_ode`` with a choice of fixed-grid solver: the whole trajectory [num_steps, B, Li, C] (grid
    points only; stage states are not returned)."""
    t = sampler_oracle.solver_grid(num_steps, x.shape[1], do_shift, time_shifting_factor, strength).to(x.device)
    kw = dict(model_kwargs)
    cond = kw.pop("cond", None)

    def f(tau, y):                                                 # velocity_ode + the output negation, transport.py:384
        t_vec = torch.ones(y.shape[0]).to(y.device) * tau          # integrators.py:109
        t_flux = torch.ones_like(t_vec) * (1 - t_vec)              # transport.py:384
        inp = y if cond is None else torch.cat((y, cond), dim=-1)  # transport.py:194-196
        return -model_fn(inp, timesteps=t_flux, **kw)

    return odeint(f, x, t, method=method)
