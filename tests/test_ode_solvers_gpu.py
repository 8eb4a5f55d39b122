"""The fixed-grid midpoint and rk4 solvers on the H100: the stage kernel against the eager torch expressions bit for bit, the
sampler against the oracle restatement with a deterministic foreign model bit for bit, the native engine path at reduced size, its
compositions with the first-block cache and both LoRA modes, the pipeline's two solves, and a full-size cfg B midpoint solve against
the unmodified reference ``transport`` on the fixed-grid ``odeint`` of ``tests/ode_oracle.py``, which is also the sampler oracle
here.  Full-size numbers are printed and kept as JSON in $VCB_REPORT_DIR (default: the system's temporary directory)."""
import dataclasses
import json
import os
import tempfile

import pytest
import torch

from conftest import GOLDEN, rel_l2

pytestmark = pytest.mark.gpu
BF16 = torch.bfloat16
STAGES = {"euler": 1, "midpoint": 2, "rk4": 4}


@pytest.fixture(scope="module", autouse=True)
def _gpu():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")


def _load(name):
    return torch.load(os.path.join(GOLDEN, name), weights_only=False)


def _cuda(d):
    return {k: (v.cuda() if torch.is_tensor(v) else v) for k, v in d.items()}


def _sampler(method, **kw):
    import visualcloze_b200.transport as T
    return T.Sampler(T.create_transport("Linear", "velocity", do_shift=True)).sample_ode(
        sampling_method=method, atol=1e-6, rtol=1e-3, reverse=False, **kw)


# ------------------------------------------------------------------------------------------------
# 1. the stage kernel is the torch expression, bit for bit
# ------------------------------------------------------------------------------------------------
def _torch_stage(method, stage, y0, vs, dt):
    """What torchdiffeq computes, with y0 and k_i = -v_i bf16 tensors and dt a 0-dim fp32 tensor on the same device."""
    k = [-v for v in vs]
    if method == "euler":
        return y0 + dt * k[0]
    if method == "midpoint":
        half_dt = 0.5 * dt
        return y0 + k[0] * half_dt if stage == 0 else y0 + dt * k[1]
    _one_third = 1 / 3
    if stage == 0:
        return y0 + dt * k[0] * _one_third
    if stage == 1:
        return y0 + dt * (k[1] - k[0] * _one_third)
    if stage == 2:
        return y0 + dt * (k[0] - k[1] + k[2])
    return y0 + (k[0] + 3 * (k[1] + k[2]) + k[3]) * dt * 0.125


def _spread(shape, g):
    """bf16 values over many binades (2^-24 .. 2^12) and both signs."""
    mant = torch.randn(shape, generator=g, device="cuda")
    expo = torch.randint(-24, 12, shape, generator=g, device="cuda").float()
    return (mant * torch.exp2(expo)).to(BF16)


def _real_dts():
    from oracle import sampler_oracle as so
    dts = []
    for N, kw in ((15, dict(do_shift=True, time_shifting_factor=1)), (8, dict(do_shift=True, time_shifting_factor=1)),
                  (31, dict(do_shift=True, time_shifting_factor=1)), (5, dict(do_shift=False, strength=0.4))):
        t = so.solver_grid(N, 3968, **kw)
        dts += [t[k + 1] - t[k] for k in range(N - 1)]
    return dts


@pytest.mark.parametrize("method,stage", [("euler", 0), ("midpoint", 0), ("midpoint", 1), ("rk4", 0), ("rk4", 1), ("rk4", 2),
                                          ("rk4", 3)])
@pytest.mark.parametrize("C,Cc", [(64, 320), (12, 5)])            # 16-byte path; the any-layout path
def test_stage_kernel_is_the_torch_expression_bitwise(method, stage, C, Cc):
    from visualcloze_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(17 * stage + C)
    rows = 2 * 333
    dts = _real_dts()
    worst = 0.0
    for i, dt in enumerate(dts[:: max(1, len(dts) // 12)]):
        y0 = _spread((rows, C), g)
        vs = [_spread((rows, C), g) for _ in range(stage + 1)]
        model_in = torch.randn(rows, C + Cc, generator=g, device="cuda").to(BF16)
        cond = model_in[:, C:].clone()
        y_out = torch.full((rows, C), float("nan"), dtype=BF16, device="cuda")
        ops.ode_stage(method, stage, y0, vs, float(dt), y_out, model_in)
        want = _torch_stage(method, stage, y0, vs, dt.cuda())
        assert want.dtype == BF16
        diff = (y_out.float() - want.float()).abs()
        fin = torch.isfinite(want.float())
        assert torch.equal(torch.isfinite(y_out.float()), fin)
        worst = max(worst, float(diff[fin].max()))
        assert torch.equal(model_in[:, :C], y_out) and torch.equal(model_in[:, C:], cond)
    assert worst == 0.0, f"{method} stage {stage}: max |diff| {worst}"


def test_euler_update_is_the_euler_stage():
    from visualcloze_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(3)
    y0, v = _spread((999, 64), g), _spread((999, 64), g)
    for dt in _real_dts()[:6]:
        a = torch.empty_like(y0)
        b = torch.empty_like(y0)
        ops.euler_update(y0, v, float(dt.to(BF16)), a)
        ops.ode_stage("euler", 0, y0, [v], float(dt), b)
        assert torch.equal(a, b) and torch.equal(a, y0 + dt.cuda() * (-v))


# ------------------------------------------------------------------------------------------------
# 2. the sampler with a deterministic foreign model is the oracle, bit for bit
# ------------------------------------------------------------------------------------------------
def _foreign(inp, timesteps, **kw):
    C = 64
    x, c = inp[..., :C], inp[..., C:]
    tt = timesteps.to(inp.dtype)[:, None, None]
    return torch.sin(3 * x) * tt + kw["scale"] * c[..., :C] - x * (1 - tt) + 0.25 * c[..., C:2 * C]


@pytest.mark.parametrize("method", ["euler", "midpoint", "rk4"])
@pytest.mark.parametrize("kw", [dict(num_steps=6, do_shift=True, time_shifting_factor=1),
                                dict(num_steps=5, do_shift=False, time_shifting_factor=None),
                                dict(num_steps=5, do_shift=False, time_shifting_factor=1.0, strength=0.4)],
                         ids=["shift", "noshift", "sdedit0.4"])
def test_foreign_model_trajectory_and_times_equal_the_oracle_bitwise(method, kw):
    import ode_oracle as so
    g = torch.Generator(device="cuda").manual_seed(5)
    B, Li = 2, 136
    x = torch.randn(B, Li, 64, generator=g, device="cuda").to(BF16)
    cond = torch.randn(B, Li, 320, generator=g, device="cuda").to(BF16)
    seen_ours, seen_orc = [], []

    def spy(seen):
        def model(inp, timesteps, **k):
            seen.append(timesteps.clone())
            return _foreign(inp, timesteps, **k)
        return model
    traj = _sampler(method, **kw)(x, spy(seen_ours), dict(cond=cond, scale=0.7))
    ref = so.sample_ode(x, spy(seen_orc), dict(cond=cond, scale=0.7), num_steps=kw["num_steps"], do_shift=kw["do_shift"],
                        time_shifting_factor=kw["time_shifting_factor"], strength=kw.get("strength"), method=method)
    assert traj.shape == ref.shape == (kw["num_steps"], B, Li, 64)
    assert torch.equal(traj, ref), f"max |diff| {float((traj.float() - ref.float()).abs().max())}"
    assert len(seen_ours) == len(seen_orc) == STAGES[method] * (kw["num_steps"] - 1)
    for a, b in zip(seen_ours, seen_orc):
        assert a.dtype == b.dtype == torch.float32 and torch.equal(a.cpu(), b.cpu())


# ------------------------------------------------------------------------------------------------
# 3. native engine path at reduced size
# ------------------------------------------------------------------------------------------------
def _build(lora_mode="merged"):
    import visualcloze_b200.model as m
    from oracle import flux_oracle as fo
    g = _load("flux_small_b1.pt")
    cfg = fo.FluxConfig(**g["cfg"])
    params = fo.make_params(cfg, seed=g["param_seed"])
    fp = m.FluxParams(**{k: v for k, v in g["cfg"].items() if k not in ("lora_rank", "lora_scale")})
    with torch.device("cuda"):
        model = m.FluxLoraWrapper(lora_rank=cfg.lora_rank, params=fp)
    model.load_state_dict({k: v.cuda() for k, v in params.items()}, strict=True)
    model.set_lora_mode(lora_mode)
    return cfg, params, model


@pytest.fixture(scope="module")
def small():
    return _build()


def _solve(model, gs, method, prepares=None):
    eng = model.engine()
    if prepares is not None:
        prep = eng.prepare

        def rec(**k):
            prepares.append(tuple(k["timesteps"].shape))
            return prep(**k)
        eng.prepare = rec
    try:
        fn = _sampler(method, **gs["kwargs"])
        return fn(gs["x"].cuda(), model.forward, dict(_cuda(gs["inputs"]), cond=gs["cond"].cuda()))
    finally:
        eng.__dict__.pop("prepare", None)


@pytest.mark.parametrize("method", ["midpoint", "rk4"])
@pytest.mark.parametrize("tag", ["shift4", "sdedit5"])
def test_native_small_vs_oracle_and_foreign_path(small, method, tag):
    import ode_oracle as so
    from oracle import flux_oracle as fo
    cfg, params, model = small
    gs = _load("sampler.pt")[tag]
    kw = gs["kwargs"]
    prepares = []
    traj = _solve(model, gs, method, prepares).cpu()
    N = kw["num_steps"]
    assert prepares == [(STAGES[method] * (N - 1), 1)], prepares
    assert traj.shape == gs["traj"].shape and torch.equal(traj[0], gs["x"])

    def model_fn(x, timesteps, **k):
        return fo.flux_forward(params, cfg, img=x, timesteps=timesteps, **k, mode="cuda_bf16")
    ref = so.sample_ode(gs["x"], model_fn, dict(gs["inputs"], cond=gs["cond"]), num_steps=N, do_shift=kw["do_shift"],
                        time_shifting_factor=kw["time_shifting_factor"], strength=kw.get("strength"), method=method)
    e_final, e_first = rel_l2(traj[-1], ref[-1]), rel_l2(traj[1], ref[1])
    print(f"[ode] {method} {tag}: final {e_final:.3e}, first interval {e_first:.3e}")
    assert e_final < 5e-2 and e_first < 1e-2, (e_final, e_first)

    calls = []

    def foreign(x, timesteps, **k):
        calls.append(float(timesteps[0]))
        return model(x, timesteps=timesteps, **k)
    traj2 = _sampler(method, **kw)(gs["x"].cuda(), foreign, dict(_cuda(gs["inputs"]), cond=gs["cond"].cuda())).cpu()
    assert len(calls) == STAGES[method] * (N - 1)
    assert rel_l2(traj2[-1], traj[-1]) < 1e-2


# ------------------------------------------------------------------------------------------------
# 4. compositions
# ------------------------------------------------------------------------------------------------
def test_first_block_cache_with_midpoint(small):
    _, _, model = small
    gs = _load("sampler.pt")["shift4"]
    plain = _solve(model, gs, "midpoint")
    try:
        model.enable_first_block_cache(0.5)
        _solve(model, gs, "midpoint")                       # one solve with the cache on, then threshold 0 = off
        st = model.cache_stats()
        E = STAGES["midpoint"] * (gs["kwargs"]["num_steps"] - 1)
        assert st["computed"] + st["skipped"] == E and st["computed"] >= 1, st
        model.enable_first_block_cache(1e30)                # skips every evaluation after the first of the solve
        _solve(model, gs, "midpoint")
        st = model.cache_stats()
        assert (st["computed"], st["skipped"]) == (1, E - 1), st
        model.enable_first_block_cache(0)
        assert torch.equal(_solve(model, gs, "midpoint"), plain)
    finally:
        model.enable_first_block_cache(None)


def test_unmerged_lora_with_midpoint(small):
    _, _, merged = small
    _, _, unmerged = _build("unmerged")
    gs = _load("sampler.pt")["shift4"]
    a, b = _solve(merged, gs, "midpoint"), _solve(unmerged, gs, "midpoint")
    e = rel_l2(b[-1].cpu(), a[-1].cpu())
    print(f"[ode] midpoint unmerged vs merged LoRA: {e:.3e}")
    assert e < 1e-2


# ------------------------------------------------------------------------------------------------
# 5. the pipeline honours `solver` in both of its solves
# ------------------------------------------------------------------------------------------------
def test_pipeline_midpoint_both_solves(small):
    from PIL import Image
    from visualcloze_b200 import pipeline as P, vae as V
    _, _, model = small
    dec = V.AutoEncoderDecoder(V.AutoEncoderParams(ch=64, ch_mult=[1, 2, 2, 2], num_res_blocks=1), device="cuda").init_synthetic(1)
    t5 = lambda prompts: (0.3 * torch.randn(len(prompts), 24, 64, generator=torch.Generator().manual_seed(len(prompts[0])))).to(BF16).cuda()
    clip = lambda prompts: torch.randn(len(prompts), 32, generator=torch.Generator().manual_seed(7)).to(BF16).cuda()

    def encode(x):
        gg = torch.Generator(device="cuda").manual_seed(int(x.shape[-1]))
        return torch.randn(x.shape[0], 16, x.shape[2] // 8, x.shape[3] // 8, generator=gg, device="cuda")

    pipe = P.VisualClozeModel(None, resolution=64, model=model, ae_decoder=dec, t5=t5, clip=clip, encode=encode, solver="midpoint")
    pipe.set_grid_size(2, 3)
    solves = []
    make = pipe._make_sample_fn

    def wrapped(num_steps, do_shift, tsf, strength):
        fn = make(num_steps, do_shift, tsf, strength)

        def spy(x, mdl, kw):
            traj = fn(x, mdl, kw)
            solves.append(dict(num_steps=num_steps, do_shift=do_shift, tsf=tsf, strength=strength, x=x.clone(),
                               kw={k: (v.clone() if torch.is_tensor(v) else v) for k, v in kw.items()}, traj=traj.clone()))
            return traj
        return spy
    pipe._make_sample_fn = wrapped
    mk = lambda: [[Image.new("RGB", (90, 90), (40 * i, 60 * j, 128)) for j in range(3)] for i in range(2)]
    imgs = mk(); imgs[1][2] = None
    up = pipe.process_images(imgs, ["layout", "task", "The last image of the last row depicts: a cat"], seed=5, cfg=30, steps=4,
                             upsampling_steps=3, upsampling_noise=0.4, is_upsampling=True)
    assert len(up) == 1 and up[0].size == (80, 80)
    assert [(s["num_steps"], s["strength"]) for s in solves] == [(4, None), (3, 0.4)]
    for s in solves:                  # each solve is the midpoint sampler run by hand on what the pipeline handed it
        assert s["traj"].shape[0] == s["num_steps"]
        fn = _sampler("midpoint", num_steps=s["num_steps"], do_shift=s["do_shift"], time_shifting_factor=s["tsf"],
                      strength=s["strength"])
        assert torch.equal(fn(s["x"], model.forward, s["kw"]), s["traj"])
        eul = _sampler("euler", num_steps=s["num_steps"], do_shift=s["do_shift"], time_shifting_factor=s["tsf"],
                       strength=s["strength"])
        assert not torch.equal(eul(s["x"], model.forward, s["kw"]), s["traj"])
    # the decoded image is the hand-run sampler's latent through the same decoder: a second run from the same seed agrees
    imgs = mk(); imgs[1][2] = None
    up2 = pipe.process_images(imgs, ["layout", "task", "The last image of the last row depicts: a cat"], seed=5, cfg=30, steps=4,
                              upsampling_steps=3, upsampling_noise=0.4, is_upsampling=True)
    assert list(up[0].getdata()) == list(up2[0].getdata())


# ------------------------------------------------------------------------------------------------
# 6. full size, cfg B: midpoint with 15 points against the reference transport on the stand-in
# ------------------------------------------------------------------------------------------------
REPORT = os.path.join(os.environ.get("VCB_REPORT_DIR") or tempfile.gettempdir(), "ode_solvers_fullsize.json")


def _record(key, **vals):
    os.makedirs(os.path.dirname(REPORT), exist_ok=True)
    data = json.load(open(REPORT)) if os.path.exists(REPORT) else {}
    data[key] = {k: float(v) for k, v in vals.items()}
    json.dump(data, open(REPORT, "w"), indent=1, sort_keys=True)
    print(f"[ode fullsize] {key}: " + ", ".join(f"{k}={v:.3e}" for k, v in vals.items()))


def test_fullsize_cfgB_midpoint_15_points_vs_reference_transport(monkeypatch):
    import ode_oracle as so
    from oracle import flux_oracle as fo, ref_runner as rr
    if not rr.available():
        pytest.skip("oracle/_ref absent")
    import bench
    import visualcloze_b200.model as M
    from test_fullsize_gpu import _MergedView
    P = M.flux_dev_fill_params()
    with torch.device("cuda"):
        ours = M.FluxLoraWrapper(lora_rank=256, params=P)
    ours.init_synthetic(0)
    sd = dict(ours.state_dict())
    ref_model = rr.build_flux(dataclasses.asdict(P), 256, sd)
    x, kw, Li, Lt = bench.make_inputs("B", 1234)
    xg, kwg = x.cuda(), _cuda(kw)
    N = 15
    traj = _sampler("midpoint", num_steps=N, do_shift=True, time_shifting_factor=1)(xg, ours.forward, kwg).float()
    assert traj.shape == (N, 1, Li, 64) and torch.isfinite(traj).all()
    _, _, _, ref_transport = rr._import()
    import transport.integrators as ref_integrators          # the unmodified reference sampler on the test's fixed-grid odeint
    monkeypatch.setattr(ref_integrators, "odeint", so.odeint)
    fn = ref_transport.Sampler(ref_transport.create_transport("Linear", "velocity", do_shift=True)).sample_ode(
        sampling_method="midpoint", num_steps=N, atol=1e-6, rtol=1e-3, reverse=False, do_shift=True, time_shifting_factor=1)
    with torch.no_grad(), torch.autocast("cuda", dtype=BF16):
        ref = fn(xg, ref_model.forward, dict(kwg)).float()
    cfg = fo.FluxConfig(**dataclasses.asdict(P), lora_rank=256)
    merged = _MergedView(sd)

    def merged_fn(inp, timesteps, **k):
        return fo.flux_forward(merged, cfg, img=inp, timesteps=timesteps.cuda(), **k, mode="cuda_bf16")
    orc = so.sample_ode(xg, merged_fn, kwg, num_steps=N, do_shift=True, time_shifting_factor=1, method="midpoint").float()
    res = dict(final_vs_reference=rel_l2(traj[-1], ref[-1]), floor_merged_oracle_vs_reference=rel_l2(orc[-1], ref[-1]),
               final_vs_merged_oracle=rel_l2(traj[-1], orc[-1]), first_interval_vs_reference=rel_l2(traj[1], ref[1]))
    _record("cfgB_midpoint_15points_28eval", **res)
    assert res["final_vs_reference"] < max(5e-2, 1.5 * res["floor_merged_oracle_vs_reference"]), res
