"""CPU checks of the fixed-grid midpoint and rk4 solvers: the sampler's method validation, the host stage-time tables against
torch's fp32 expressions, the test oracle (``tests/ode_oracle.py``) against the expressions written out, the pinned Euler oracle,
the Euler stand-in and the unmodified reference ``transport`` driving it (when ``oracle/_ref`` is present), its convergence
orders, and the C ABI of ``vcb_ode_stage``."""
import ctypes as C
import math
import os
import re
import sys
import types

import pytest
import torch

from conftest import REPO

BF16 = torch.bfloat16


def _sampler():
    from visualcloze_b200 import transport as T
    return T.Sampler(T.create_transport("Linear", "velocity", do_shift=True))


@pytest.mark.parametrize("method", ["dopri5", "bosh3", "adaptive_heun", "heun2", "heun3", "explicit_adams", "implicit_adams",
                                    "fixed_adams", "dopri8", "RK4", None])
def test_unsupported_methods_raise_and_name_the_supported_set(method):
    with pytest.raises(NotImplementedError) as e:
        _sampler().sample_ode(sampling_method=method, num_steps=4)
    assert all(f"'{m}'" in str(e.value) for m in ("euler", "midpoint", "rk4")), str(e.value)


@pytest.mark.parametrize("method", ["euler", "midpoint", "rk4"])
def test_supported_methods_return_a_callable(method):
    assert callable(_sampler().sample_ode(sampling_method=method, num_steps=4, do_shift=True, time_shifting_factor=1))


def _torchdiffeq_stage_times(t, method):
    """The evaluation times as torchdiffeq forms them, interval by interval on 0-dim fp32 tensors."""
    out = []
    for k in range(len(t) - 1):
        t0, t1 = t[k], t[k + 1]
        dt = t1 - t0
        if method == "euler":
            row = [t0]
        elif method == "midpoint":
            half_dt = 0.5 * dt
            row = [t0, t0 + half_dt]
        else:
            row = [t0, t0 + dt * (1 / 3), t0 + dt * (2 / 3), t1]
        out.append(torch.stack(row))
    return torch.stack(out)


@pytest.mark.parametrize("method", ["euler", "midpoint", "rk4"])
@pytest.mark.parametrize("do_shift,tsf,strength", [(True, 1, None), (False, None, None), (True, 3.0, None), (False, 1, None),
                                                   (True, 1, 0.4), (False, None, 0.4)])
def test_stage_time_tables_equal_torch_fp32_expressions(method, do_shift, tsf, strength):
    from oracle import sampler_oracle as so
    from visualcloze_b200 import transport as T
    N, Li = 15, 3968
    t0 = 0.0 if strength is None else strength
    t = T.solver_grid(t0, 1.0, N, Li, do_shift, tsf)
    assert torch.equal(t, so.solver_grid(N, Li, do_shift, tsf, strength))
    got = T.stage_times(t, method)
    want = _torchdiffeq_stage_times(t, method)
    assert got.dtype == torch.float32 and got.shape == (N - 1, {"euler": 1, "midpoint": 2, "rk4": 4}[method])
    assert torch.equal(got, want)
    # what the model is handed: 1 - bf16(tau) (the _PerturbFunc cast), evaluation e = k * stages + s
    flux = 1 - got.reshape(-1).to(BF16).float()
    assert torch.equal(flux, torch.stack([1 - tau.to(BF16).float() for tau in want.reshape(-1)]))
    if method == "rk4":
        assert torch.equal(got[:, 3], t[1:]) and torch.equal(got[:-1, 3], got[1:, 0])


# ---- the test oracle (tests/ode_oracle.py) -------------------------------------------------------------------------------------
def _toy_model(inp, timesteps, scale):
    """Pure elementwise, deterministic: depends on the state, on cond and on the time the model is handed."""
    C = 8
    x, c = inp[..., :C], inp[..., C:]
    tt = timesteps.to(inp.dtype)[:, None, None]
    return torch.sin(3 * x) * tt + scale * c[..., :C] - x * (1 - tt) + 0.25


def _toy_inputs(B=2, L=24, C=8, Cc=16, seed=0):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, L, C, generator=g).to(BF16)
    cond = (0.5 * torch.randn(B, L, Cc, generator=g)).to(BF16)
    return x, cond


def _written_out(x, model_fn, cond, method, N, do_shift, tsf, strength):
    """The torchdiffeq expressions written out once more, interval by interval, independently of ode_oracle's step table."""
    from oracle import sampler_oracle as so
    t = so.solver_grid(N, x.shape[1], do_shift, tsf, strength)

    def f(tau, y):
        tv = torch.ones(y.shape[0]) * tau.to(y.dtype)
        return -model_fn(torch.cat((y, cond), dim=-1), timesteps=torch.ones_like(tv) * (1 - tv))
    ys, y = [x], x
    for k in range(N - 1):
        t0, t1 = t[k], t[k + 1]
        dt = t1 - t0
        if method == "euler":
            y = y + dt * f(t0, y)
        elif method == "midpoint":
            half_dt = 0.5 * dt
            k1 = f(t0, y)
            y = y + dt * f(t0 + half_dt, y + k1 * half_dt)
        else:
            k1 = f(t0, y)
            k2 = f(t0 + dt * (1 / 3), y + dt * k1 * (1 / 3))
            k3 = f(t0 + dt * (2 / 3), y + dt * (k2 - k1 * (1 / 3)))
            k4 = f(t1, y + dt * (k1 - k2 + k3))
            y = y + (k1 + 3 * (k2 + k3) + k4) * dt * 0.125
        ys.append(y)
    return torch.stack(ys)


@pytest.mark.parametrize("method", ["euler", "midpoint", "rk4"])
@pytest.mark.parametrize("do_shift,tsf,strength", [(True, 1, None), (False, None, None), (True, 1, 0.4)])
def test_test_oracle_is_the_written_out_expressions_bitwise_bf16(method, do_shift, tsf, strength):
    import ode_oracle
    from oracle import sampler_oracle as so
    x, cond = _toy_inputs()
    N = 6
    model = lambda inp, timesteps: _toy_model(inp, timesteps, 0.7)
    got = ode_oracle.sample_ode(x, model, {"cond": cond}, num_steps=N, do_shift=do_shift, time_shifting_factor=tsf,
                                strength=strength, method=method)
    assert got.dtype == BF16 and got.shape == (N, *x.shape)
    assert torch.equal(got, _written_out(x, model, cond, method, N, do_shift, tsf, strength))
    eul = so.sample_ode(x, model, {"cond": cond}, num_steps=N, do_shift=do_shift, time_shifting_factor=tsf, strength=strength)
    if method == "euler":                  # the pinned Euler oracle, bit for bit
        assert torch.equal(got, eul)
    else:
        assert not torch.equal(got[-1], eul[-1])


def test_test_oracle_euler_is_the_stand_in_bitwise():
    """On Euler, ode_oracle.odeint is the stand-in oracle/build_ref.py writes, bit for bit."""
    import ode_oracle
    from oracle import build_ref
    stand_in = types.ModuleType("torchdiffeq_stand_in")
    exec(compile(build_ref._TORCHDIFFEQ, "torchdiffeq_stand_in", "exec"), stand_in.__dict__)
    x, cond = _toy_inputs(seed=1)
    t = torch.linspace(0.2, 1.0, 7)

    def f(tau, y):
        return -_toy_model(torch.cat((y, cond), dim=-1), 1 - torch.ones(y.shape[0]) * tau, 0.3)
    assert torch.equal(ode_oracle.odeint(f, x, t, method="euler"), stand_in.odeint(f, x, t, method="euler"))


@pytest.mark.parametrize("method", ["midpoint", "rk4"])
def test_unmodified_reference_transport_drives_the_test_oracle(method, monkeypatch):
    """The reference's own Sampler (transport/*.py, unmodified, from oracle/_ref) with ode_oracle.odeint as its torchdiffeq."""
    import ode_oracle
    from oracle import build_ref, ref_runner
    if not ref_runner.available():
        pytest.skip("oracle/_ref absent")
    build_ref.verify()
    for entry in (ref_runner.REF, ref_runner.ARCHIVE):
        if entry not in sys.path:
            sys.path.insert(0, entry)
    import transport as ref_transport
    import transport.integrators as ref_integrators
    monkeypatch.setattr(ref_integrators, "odeint", ode_oracle.odeint)
    x, cond = _toy_inputs(seed=3)
    seen = []

    def model(inp, timesteps, **kw):
        seen.append(timesteps.clone())
        return _toy_model(inp, timesteps, kw["scale"])
    for kw in (dict(do_shift=True, time_shifting_factor=1), dict(do_shift=False, time_shifting_factor=None, strength=0.4)):
        fn = ref_transport.Sampler(ref_transport.create_transport("Linear", "velocity", do_shift=True)).sample_ode(
            sampling_method=method, num_steps=5, atol=1e-6, rtol=1e-3, reverse=False, **kw)
        seen.clear()
        ref = fn(x, model, dict(cond=cond, scale=0.7))
        n_ref = len(seen)
        got = ode_oracle.sample_ode(x, model, dict(cond=cond, scale=0.7), num_steps=5, do_shift=kw["do_shift"],
                                    time_shifting_factor=kw["time_shifting_factor"], strength=kw.get("strength"), method=method)
        assert torch.equal(got, ref)
        assert n_ref == {"midpoint": 2, "rk4": 4}[method] * 4
        assert all(torch.equal(a, b) for a, b in zip(seen[:n_ref], seen[n_ref:]))


def _oracle_solve(y0, method, N, lam):
    import ode_oracle
    return ode_oracle.sample_ode(y0, lambda inp, timesteps: -lam * inp, {}, num_steps=N, do_shift=False, method=method)


def _odeint_solve(y0, method, N, lam):
    import ode_oracle
    return ode_oracle.odeint(lambda tau, y: lam * y, y0, torch.linspace(0.0, 1.0, N), method=method)


@pytest.mark.parametrize("solve", [_oracle_solve, _odeint_solve], ids=["sample_ode", "odeint"])
@pytest.mark.parametrize("method,order", [("euler", 1), ("midpoint", 2), ("rk4", 4)])
def test_convergence_order_float64(solve, method, order):
    lam = -1.3
    errs = []
    for n in (5, 9, 17, 33):
        traj = solve(torch.ones(1, 1, 4, dtype=torch.float64), method, n, lam)
        errs.append(float((traj[-1] - math.exp(lam)).abs().max()))          # dy/dtau = lam * y on tau in [0, 1]
    orders = [math.log2(a / b) for a, b in zip(errs, errs[1:])]
    assert all(abs(o - order) < 0.25 for o in orders), (errs, orders)


def test_convergence_order_float64_time_dependent():
    """dy/dtau = cos(tau) y: a wrong stage time would spoil the order where the autonomous problem cannot see it."""
    import ode_oracle
    exact = math.exp(math.sin(1.0))
    for method, order in (("midpoint", 2), ("rk4", 4)):
        errs = []
        for n in (17, 33, 65):
            y0 = torch.ones(1, 1, 2, dtype=torch.float64)
            traj = ode_oracle.sample_ode(y0, lambda inp, timesteps: -torch.cos(1 - timesteps.double())[:, None, None] * inp, {},
                                         num_steps=n, do_shift=False, method=method)
            errs.append(float((traj[-1] - exact).abs().max()))
        orders = [math.log2(a / b) for a, b in zip(errs, errs[1:])]
        assert all(abs(o - order) < 0.2 for o in orders), (method, errs, orders)


def test_ctypes_prototype_and_abi_7():
    from visualcloze_b200 import _lib, ops
    assert _lib._SIGNATURES["vcb_ode_stage"] == (C.c_int, [C.c_int32, C.c_int32, C.c_void_p, C.POINTER(C.c_void_p), C.c_int32,
                                                          C.c_float, C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_int32,
                                                          C.c_void_p])
    header = open(os.path.join(REPO, "include", "vcb200.h")).read()
    assert re.search(r"int vcb_ode_stage\(int32_t method, int32_t stage, const void\* y0, const void\* const\* v, int32_t n_v, "
                     r"float dt,\s+void\* y_out, void\* model_in, int64_t ld_in, int64_t rows, int32_t C, void\* stream\);", header)
    for name, val in ops.ODE_METHODS.items():
        assert int(re.search(rf"#define VCB_ODE_{name.upper()} (\d+)", header).group(1)) == val
    assert int(re.search(r"#define VCB_ABI_VERSION (\d+)", header).group(1)) == 7
    lib = _lib.lib()
    assert lib.vcb_abi_version() == 7 and _lib.ABI_VERSION == 7
    assert lib.vcb_ode_stage.restype is C.c_int


@pytest.mark.parametrize("method,stage,n_v", [(3, 0, 1), (-1, 0, 1), (0, 1, 2), (1, 2, 3), (2, 4, 5), (2, 1, 1), (1, 1, 1),
                                              (0, 0, 2)])
def test_c_refuses_bad_method_stage_and_output_count(method, stage, n_v):
    """Argument checks run before any device work, so they are exercised without a GPU."""
    from visualcloze_b200 import _lib
    lib = _lib.lib()
    ptrs = (C.c_void_p * 5)(*([256] * 5))
    assert lib.vcb_ode_stage(method, stage, C.c_void_p(256), ptrs, n_v, 0.1, C.c_void_p(512), None, 0, 4, 8, None) != 0
    assert lib.vcb_last_error().startswith(b"ode_stage:")
    ptrs[0] = None
    assert lib.vcb_ode_stage(0, 0, C.c_void_p(256), ptrs, 1, 0.1, C.c_void_p(512), None, 0, 4, 8, None) != 0
    assert lib.vcb_ode_stage(0, 0, C.c_void_p(256), (C.c_void_p * 1)(256), 1, 0.1, C.c_void_p(512), C.c_void_p(768), 4, 4, 8,
                             None) != 0
    assert b"ld_in" in lib.vcb_last_error()
