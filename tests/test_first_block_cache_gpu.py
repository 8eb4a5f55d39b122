"""The opt-in first-block cache on the H100: off is bitwise the plain engine, a repeated evaluation is reused exactly, the skip
decisions and per-step diffs follow a test-local FBCache over the restated oracle, right padding is excluded, prepare resets the
cache, and (recorded, not judged) what it does at full size over 29 evaluations.

The cache is NOT the reference's numerics; the only bar against the oracle is the trajectory bar of test_flux_gpu.py (5e-2)."""
import dataclasses
import json
import math
import os
import tempfile

import pytest
import torch

from conftest import GOLDEN, rel_l2

pytestmark = pytest.mark.gpu
BF16 = torch.bfloat16


@pytest.fixture(scope="module", autouse=True)
def _gpu():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")


def _load(name):
    return torch.load(os.path.join(GOLDEN, name), weights_only=False)


def _cuda(d):
    return {k: (v.cuda() if torch.is_tensor(v) else v) for k, v in d.items()}


def _build(cfg_dict, seed, lora_mode="merged", precision="bf16", threshold=None):
    import visualcloze_b200.model as m
    from oracle import flux_oracle as fo
    cfg = fo.FluxConfig(**cfg_dict)
    params = fo.make_params(cfg, seed=seed)
    fp = m.FluxParams(**{k: v for k, v in cfg_dict.items() if k not in ("lora_rank", "lora_scale")})
    with torch.device("cuda"):
        model = m.FluxLoraWrapper(lora_rank=cfg.lora_rank, params=fp)
    model.load_state_dict({k: v.cuda() for k, v in params.items()}, strict=True)
    model.set_lora_mode(lora_mode)
    model.set_linear_precision(precision)
    model.enable_first_block_cache(threshold)
    return cfg, params, model


def _prepare(model, inp, E):
    """engine.prepare for E evaluations at the input's time (one solve)."""
    eng = model.engine()
    eng.prepare(txt=inp["txt"], y=inp["y"], img_ids=inp["img_ids"], txt_ids=inp["txt_ids"],
                timesteps=inp["timesteps"][None].expand(E, -1).contiguous(), guidance=inp["guidance"], txt_mask=inp["txt_mask"],
                img_mask=inp["img_mask"], n_img_tokens=inp["img"].shape[1])
    return eng


def _sample(model, gs, num_steps, record=None):
    """The Euler sampler through the public API (native engine path); `record` receives cache_stats() after every evaluation."""
    import visualcloze_b200.transport as t
    eng = model.engine()
    if record is not None:
        fwd = eng.forward

        def rec(*a, **k):
            out = fwd(*a, **k)
            record.append(eng.cache_stats())
            return out
        eng.forward = rec
    try:
        fn = t.Sampler(t.create_transport("Linear", "velocity", do_shift=True)).sample_ode(
            sampling_method="euler", num_steps=num_steps, atol=1e-6, rtol=1e-3, reverse=False, do_shift=True, time_shifting_factor=1)
        return fn(gs["x"].cuda(), model.forward, dict(_cuda(gs["inputs"]), cond=gs["cond"].cuda()))
    finally:
        eng.__dict__.pop("forward", None)


# ------------------------------------------------------------------------------------------------
# 1. off is identical
# ------------------------------------------------------------------------------------------------
def test_threshold_zero_is_bitwise_the_plain_engine():
    g, gs = _load("flux_small_b1.pt"), _load("sampler.pt")["shift4"]
    _, _, plain = _build(g["cfg"], g["param_seed"])
    _, _, toggled = _build(g["cfg"], g["param_seed"], threshold=0.5)
    inp = _cuda(g["inputs"])
    assert toggled(**inp).shape == plain(**inp).shape          # one run with the cache on
    toggled.enable_first_block_cache(0)
    assert torch.equal(toggled(**inp), plain(**inp))
    assert torch.equal(_sample(toggled, gs, 4), _sample(plain, gs, 4))
    toggled.enable_first_block_cache(None)
    assert torch.equal(_sample(toggled, gs, 4), _sample(plain, gs, 4))


# ------------------------------------------------------------------------------------------------
# 2. exact reuse
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", ["merged_bf16", "unmerged", "fp8"])
def test_repeated_evaluation_is_skipped_and_bitwise(mode):
    """Two forwards with the same eval index and input: the second is skipped with diff 0 and returns exactly the first's output.
    Bitwise because R = x_final - x1 is exact in fp32 (so bf16(x1 + R) == x_final) and, with the cache on, the final LayerNorm
    computes its row statistics itself on computed and skipped evaluations alike."""
    g = _load("flux_small_b1.pt")
    kw = dict(merged_bf16={}, unmerged=dict(lora_mode="unmerged"), fp8=dict(precision="fp8"))[mode]
    _, _, model = _build(g["cfg"], g["param_seed"], threshold=1e-3, **kw)
    inp = _cuda(g["inputs"])
    eng = _prepare(model, inp, 1)
    out1 = eng.forward(0, inp["img"]).clone()
    s1 = eng.cache_stats()
    assert (s1["computed"], s1["skipped"]) == (1, 0) and s1["last_diff"] == math.inf
    out2 = eng.forward(0, inp["img"])
    s2 = eng.cache_stats()
    assert (s2["computed"], s2["skipped"]) == (1, 1) and s2["last_diff"] == 0.0, s2
    print(f"[first_block_cache] {mode}: the skipped evaluation is bitwise the computed one (final LayerNorm statistics "
          "computed by the LayerNorm kernel on both)")
    assert torch.equal(out1, out2)
    # the cached residual is that of the last COMPUTED evaluation: a third call is reused again, still exactly
    assert torch.equal(eng.forward(0, inp["img"]), out1) and eng.cache_stats()["skipped"] == 2


# ------------------------------------------------------------------------------------------------
# 3. decisions against an FBCache over the restated oracle
# ------------------------------------------------------------------------------------------------
class _OracleFBCache:
    """FBCache (ParaAttention / diffusers FirstBlockCache) over oracle/flux_oracle.py, with the engine's definitions: r = bf16(x1 -
    x0) over the img rows, diff = sum|r - r_ref| / sum|r_ref| over the valid rows, R = x_final - x1 in fp32."""

    def __init__(self, fo, params, cfg, threshold):
        self.fo, self.p, self.cfg, self.t = fo, params, cfg, threshold
        self.k, self.r_ref, self.R = 0, None, None
        self.diffs, self.skips = [], []

    def __call__(self, img, timesteps, img_ids, txt, txt_ids, y, txt_mask=None, img_mask=None, guidance=None):
        fo, p, cfg = self.fo, self.p, self.cfg
        nm, ls = fo.Numerics("cuda_bf16"), cfg.lora_scale
        x0 = fo.lora_linear(p, "img_in", img, nm, ls)
        vec = fo.flux_vec(p, cfg, timesteps, y, guidance, nm, ls)
        txt = fo.lora_linear(p, "txt_in", txt, nm, ls)
        cos, sin = fo.rope_table(torch.cat((txt_ids, img_ids), dim=1), cfg.axes_dim, cfg.theta)
        mask = torch.cat((txt_mask, img_mask), dim=1)
        x1, txt = fo.double_block(p, 0, cfg, x0, txt, vec, cos, sin, mask, nm, ls)
        r = (x1.float() - x0.float()).to(BF16).float()
        valid = img_mask.bool()[..., None].float()
        skip = False
        if self.k > 0:
            diff = float(((r - self.r_ref).abs() * valid).sum() / (self.r_ref.abs() * valid).sum())
            self.diffs.append(diff)
            skip = diff < self.t
        self.k += 1
        self.skips.append(skip)
        if skip:
            img = (x1.float() + self.R).to(BF16)
        else:
            img = x1
            for i in range(1, cfg.depth):
                img, txt = fo.double_block(p, i, cfg, img, txt, vec, cos, sin, mask, nm, ls)
            x = torch.cat((txt, img), 1)
            for i in range(cfg.depth_single_blocks):
                x = fo.single_block(p, i, cfg, x, vec, cos, sin, mask, nm, ls)
            img = x[:, txt.shape[1]:]
            self.r_ref, self.R = r, img.float() - x1.float()
        return fo.last_layer(p, img, vec, nm, ls)


def test_decisions_match_an_fbcache_over_the_oracle():
    from oracle import flux_oracle as fo
    from oracle import sampler_oracle as so
    g, gs = _load("flux_small_b1.pt"), _load("sampler.pt")["shift4"]
    cfg_dict = dict(g["cfg"], depth=2, depth_single_blocks=2)
    cfg, params, model = _build(cfg_dict, g["param_seed"])
    steps = 9

    def ours(threshold):
        model.enable_first_block_cache(threshold)
        rec = []
        traj = _sample(model, gs, steps, rec).cpu()
        diffs = [s["last_diff"] for s in rec[1:]]
        skips = [False] + [b["skipped"] > a["skipped"] for a, b in zip(rec, rec[1:])]
        return traj, diffs, skips

    def oracle(threshold):
        m = _OracleFBCache(fo, params, cfg, threshold)
        traj = so.sample_ode(gs["x"], m, dict(gs["inputs"], cond=gs["cond"]), num_steps=steps, do_shift=True, time_shifting_factor=1)
        return traj, m.diffs, m.skips

    # per-step diffs with nothing skipped (a threshold below any diff keeps the cache on)
    traj0, d_ours, s_ours = ours(1e-30)
    _, d_orc, _ = oracle(1e-30)
    assert not any(s_ours) and len(d_ours) == steps - 2
    for a, b in zip(d_ours, d_orc):
        assert abs(a - b) <= 2e-2 * b, (d_ours, d_orc)
    print("[first_block_cache] per-step diff ours / oracle: " + ", ".join(f"{a:.4g}/{b:.4g}" for a, b in zip(d_ours, d_orc)))
    # thresholds between observed diffs; a case counts when it is >= 10 % away from every diff either run observes with it
    ds = sorted(d_ours)
    candidates = [0.5 * ds[0]] + [math.sqrt(a * b) for a, b in zip(ds, ds[1:])] + [2.0 * ds[-1]]
    checked = []
    for t in candidates:
        traj, d1, s1 = ours(t)
        ref, d2, s2 = oracle(t)
        if any(abs(d - t) < 0.1 * t for d in d1 + d2):
            continue
        assert s1 == s2, (t, s1, s2, d1, d2)
        assert rel_l2(traj[-1], ref[-1]) < 5e-2, t
        checked.append((t, sum(s1)))
    print(f"[first_block_cache] (threshold, skipped) checked: {checked}")
    assert any(n > 0 for _, n in checked), (checked, d_ours)
    model.enable_first_block_cache(None)
    assert rel_l2(traj0[-1], _sample(model, gs, steps).cpu()[-1]) < 1e-2


def test_mixed_decisions_match_the_oracle_on_spread_inputs():
    """With random weights the per-step diffs of a sampler solve lie close together, so the thresholds 10 % away from all of them
    skip everything or nothing.  Here one solve's evaluations get inputs perturbed by amounts spread over three decades, which
    spreads the diffs: thresholds between them give mixed decisions, checked against the oracle's FBCache evaluation by
    evaluation."""
    from oracle import flux_oracle as fo
    g = _load("flux_small_b1.pt")
    cfg, params, model = _build(g["cfg"], g["param_seed"])
    inp = g["inputs"]
    gen = torch.Generator().manual_seed(11)
    scales = [0.0, 0.003, 1.0, 0.01, 0.3, 0.001, 3.0, 0.03]
    imgs = [(inp["img"].float() + s * torch.randn(inp["img"].shape, generator=gen)).to(BF16) for s in scales]

    def ours(threshold):
        model.enable_first_block_cache(threshold)
        eng = _prepare(model, _cuda(inp), len(imgs))
        outs, diffs, skips = [], [], []
        for k, img in enumerate(imgs):
            before = eng.cache_stats()["skipped"]
            outs.append(eng.forward(k, img.cuda()).cpu())
            st = eng.cache_stats()
            skips.append(st["skipped"] > before)
            if k:
                diffs.append(st["last_diff"])
        return outs, diffs, skips

    def oracle(threshold):
        m = _OracleFBCache(fo, params, cfg, threshold)
        kw = {k: v for k, v in inp.items() if k != "img"}
        return [m(img=img, **kw) for img in imgs], m.diffs, m.skips

    _, d_ours, _ = ours(1e-30)
    _, d_orc, _ = oracle(1e-30)
    # 2e-2 relative as in the sampler test, plus an absolute floor: the two sides round r = bf16(x1 - x0) from x1 values that
    # differ in the last bf16 bit here and there, which on the smallest diffs here (~5e-3) is a few 1e-4
    for a, b in zip(d_ours, d_orc):
        assert abs(a - b) <= 2e-2 * b + 1e-3, (d_ours, d_orc)
    ds = sorted(d_ours)
    mixed = []
    for t in [math.sqrt(a * b) for a, b in zip(ds, ds[1:]) if b > 1.5 * a]:
        o1, d1, s1 = ours(t)
        o2, d2, s2 = oracle(t)
        if any(abs(d - t) < 0.1 * t for d in d1 + d2):
            continue
        assert s1 == s2, (t, s1, s2, d1, d2)
        for a, b in zip(o1, o2):
            assert rel_l2(a, b) < 5e-2, t
        mixed.append((t, sum(s1)))
    print(f"[first_block_cache] spread inputs, diffs {[round(d, 4) for d in d_ours]}; (threshold, skipped) checked: {mixed}")
    assert any(0 < n < len(imgs) - 1 for _, n in mixed), mixed


# ------------------------------------------------------------------------------------------------
# 4. padding
# ------------------------------------------------------------------------------------------------
def test_padded_rows_change_neither_the_decision_nor_the_valid_outputs():
    g = _load("flux_small_b2r.pt")
    inp = _cuda(g["inputs"])
    assert int(inp["img_mask"].sum(-1).min()) < inp["img_mask"].shape[1], "the fixture is right-padded"
    pad = ~inp["img_mask"].bool()
    gen = torch.Generator(device="cuda").manual_seed(3)
    img_b = (inp["img"].float() + 0.05 * torch.randn(inp["img"].shape, generator=gen, device="cuda")).to(BF16)

    def garbage(x):
        noise = 300.0 * torch.randn(x.shape, generator=gen, device="cuda")
        return torch.where(pad[..., None], noise.to(BF16), x)

    for threshold in (1e-6, 1e6):                                # the second evaluation computed, then skipped
        _, _, model = _build(g["cfg"], g["param_seed"], threshold=threshold)
        runs = []
        for a, b in ((inp["img"], img_b), (garbage(inp["img"]), garbage(img_b))):
            eng = _prepare(model, inp, 2)
            o0 = eng.forward(0, a).clone()
            o1 = eng.forward(1, b).clone()
            runs.append((o0, o1, eng.cache_stats()))
        (a0, a1, sa), (b0, b1, sb) = runs
        assert sa == sb and sa["computed"] + sa["skipped"] == 2, (sa, sb)
        assert sa["skipped"] == (1 if threshold > 1 else 0) and 0 < sa["last_diff"] < math.inf
        valid = inp["img_mask"].bool()
        assert torch.equal(a0[valid], b0[valid]) and torch.equal(a1[valid], b1[valid])


# ------------------------------------------------------------------------------------------------
# 5. reset
# ------------------------------------------------------------------------------------------------
def test_prepare_resets_the_cache():
    g = _load("flux_small_b1.pt")
    _, _, model = _build(g["cfg"], g["param_seed"], threshold=1e6)
    inp = _cuda(g["inputs"])
    eng = _prepare(model, inp, 2)
    first = eng.forward(0, inp["img"]).clone()
    eng.forward(1, inp["img"])
    assert (eng.cache_stats()["computed"], eng.cache_stats()["skipped"]) == (1, 1)
    eng = _prepare(model, inp, 2)
    s = eng.cache_stats()
    assert (s["computed"], s["skipped"]) == (0, 0) and math.isnan(s["last_diff"])
    again = eng.forward(0, inp["img"])
    s = eng.cache_stats()
    assert (s["computed"], s["skipped"], s["last_diff"]) == (1, 0, math.inf)
    assert torch.equal(again, first)
    # switching the cache off and on changes the workspace layout: the engine asks for a new prepare
    model.enable_first_block_cache(None)
    model.enable_first_block_cache(0.1)
    from visualcloze_b200._lib import VcbError
    with pytest.raises(VcbError):
        eng.forward(0, inp["img"])


# ------------------------------------------------------------------------------------------------
# 6. full size, cfg B, 29 evaluations (recorded, not judged)
# ------------------------------------------------------------------------------------------------
# measured values are printed and kept as JSON in $VCB_REPORT_DIR (default: the system's temporary directory)
REPORT = os.path.join(os.environ.get("VCB_REPORT_DIR") or tempfile.gettempdir(), "first_block_cache_fullsize.json")


def _record(key, **vals):
    os.makedirs(os.path.dirname(REPORT), exist_ok=True)
    data = json.load(open(REPORT)) if os.path.exists(REPORT) else {}
    data[key] = {k: float(v) for k, v in vals.items()}
    json.dump(data, open(REPORT, "w"), indent=1, sort_keys=True)
    print(f"[first_block_cache] {key}: " + ", ".join(f"{k}={float(v):.4g}" for k, v in vals.items()))


def test_fullsize_cfgB_29_evaluations_recorded():
    import bench
    import visualcloze_b200.model as M
    import visualcloze_b200.transport as T
    from oracle import ref_runner as rr
    P = M.flux_dev_fill_params()
    with torch.device("cuda"):
        ours = M.FluxLoraWrapper(lora_rank=256, params=P)
    ours.init_synthetic(0)
    x, kw, Li, Lt = bench.make_inputs("B", 1234)
    xg, kwg = x.cuda(), _cuda(kw)
    fn = T.Sampler(T.create_transport("Linear", "velocity", do_shift=True)).sample_ode(
        sampling_method="euler", num_steps=30, atol=1e-6, rtol=1e-3, reverse=False, do_shift=True, time_shifting_factor=1)

    def run(threshold, record=None):
        ours.enable_first_block_cache(threshold)
        eng = ours.engine()
        if record is not None:
            fwd = eng.forward

            def rec(*a, **k):
                out = fwd(*a, **k)
                record.append(eng.cache_stats()["last_diff"])
                return out
            eng.forward = rec
        fn(xg, ours.forward, kwg)                                  # warm-up of this setting
        torch.cuda.synchronize()
        t0 = torch.cuda.Event(enable_timing=True)
        t1 = torch.cuda.Event(enable_timing=True)
        if record is not None:
            record.clear()
        t0.record()
        traj = fn(xg, ours.forward, kwg)
        t1.record()
        torch.cuda.synchronize()
        eng.__dict__.pop("forward", None)
        return traj[-1].float(), t0.elapsed_time(t1), eng.cache_stats()

    base, ms_off, _ = run(None)
    diffs = []
    probe, ms_probe, _ = run(1e-30, diffs)
    ds = sorted(d for d in diffs[1:] if math.isfinite(d))
    res = {"off": dict(sampler_ms=ms_off),
           "on_never_skipping": dict(sampler_ms=ms_probe, final_vs_uncached=rel_l2(probe, base), diff_min=ds[0],
                                     diff_median=ds[len(ds) // 2], diff_max=ds[-1])}
    lats = {"off": base}
    for t in (ds[len(ds) // 3], ds[2 * len(ds) // 3]):          # thresholds that skip some of the 29 evaluations
        lat, ms, st = run(t)
        assert st["computed"] + st["skipped"] == 29 and torch.isfinite(lat).all()
        key = f"threshold_{t:.4g}"
        res[key] = dict(threshold=t, computed=st["computed"], skipped=st["skipped"], sampler_ms=ms,
                        final_vs_uncached=rel_l2(lat, base))
        lats[key] = lat
    ours._engine = None                                           # room for the reference modules
    torch.cuda.empty_cache()
    if rr.available():
        refm = rr.build_flux(dataclasses.asdict(P), 256, dict(ours.state_dict()))
        ref = rr.sample_ode(refm, xg, kwg, num_steps=30, do_shift=True, time_shifting_factor=1)[-1].float()
        del refm
        for key, lat in lats.items():
            res[key]["final_vs_reference"] = rel_l2(lat, ref)
    for key, vals in res.items():
        _record(f"cfgB_29eval_{key}", **vals)
    del ours
    torch.cuda.empty_cache()
