"""Batched requests on the H100: a B = 3 solve against three B = 1 solves (reduced size) and one full-size cfg B solve at B = 2, the
per-sample first-block cache (bitwise the per-batch mode at B = 1, per-sample decisions equal to solo runs at B = 3, exact reuse,
padding excluded, per-batch mode at B > 1 untouched), and ``process_images_batch`` against solo ``process_images`` / SDEdit calls:
the noise and sampler inputs bit for bit, the images within the pipeline bound (PSNR >= 35 dB).

Measured values are printed and kept as JSON in $VCB_REPORT_DIR (default: the system's temporary directory)."""
import json
import math
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest
import torch

from conftest import GOLDEN, REPO, rel_l2

pytestmark = pytest.mark.gpu
BF16 = torch.bfloat16
REPORT = os.path.join(os.environ.get("VCB_REPORT_DIR") or tempfile.gettempdir(), "batch_requests.json")


@pytest.fixture(scope="module", autouse=True)
def _gpu():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")


def _record(key, **vals):
    os.makedirs(os.path.dirname(REPORT), exist_ok=True)
    data = json.load(open(REPORT)) if os.path.exists(REPORT) else {}
    data[key] = vals
    json.dump(data, open(REPORT, "w"), indent=1, sort_keys=True)
    print(f"[batch] {key}: {vals}")


def _load(name):
    return torch.load(os.path.join(GOLDEN, name), weights_only=False)


def _cuda(d):
    return {k: (v.cuda() if torch.is_tensor(v) else v) for k, v in d.items()}


def _build(cfg_dict, seed, lora_mode="merged", precision="bf16"):
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
    return model


def _batch_inputs(inp, B, seed=1):
    """B samples around the one-sample fixture: own img, txt, y and guidance per sample"""
    g = torch.Generator().manual_seed(seed)
    out = {}
    for k, v in inp.items():
        rep = v.expand(B, *v.shape[1:]).clone()
        if k in ("img", "txt", "y"):
            rep = (rep.float() + 0.3 * torch.randn(rep.shape, generator=g)).to(v.dtype)
        elif k == "guidance":
            rep = torch.tensor([30.0, 3.5, 10.0, 4.0][:B]).to(v.dtype)
        out[k] = rep
    return out


def _pick(d, b):
    return {k: v[b:b + 1] for k, v in d.items()}


def _prepare(model, inp, E):
    eng = model.engine()
    eng.prepare(txt=inp["txt"], y=inp["y"], img_ids=inp["img_ids"], txt_ids=inp["txt_ids"],
                timesteps=inp["timesteps"][None].expand(E, -1).contiguous(), guidance=inp["guidance"], txt_mask=inp["txt_mask"],
                img_mask=inp["img_mask"], n_img_tokens=inp["img"].shape[1])
    return eng


def _sampler(num_steps):
    import visualcloze_b200.transport as t
    return t.Sampler(t.create_transport("Linear", "velocity", do_shift=True)).sample_ode(
        sampling_method="euler", num_steps=num_steps, atol=1e-6, rtol=1e-3, reverse=False, do_shift=True, time_shifting_factor=1)


# ------------------------------------------------------------------------------------------------
# engine: batched solves against solo solves
# ------------------------------------------------------------------------------------------------
def test_b3_solve_matches_three_b1_solves():
    g = _load("flux_small_b1.pt")
    model = _build(g["cfg"], g["param_seed"])
    inp = _batch_inputs(g["inputs"], 3)
    gen = torch.Generator().manual_seed(5)
    x = torch.randn(3, inp["img"].shape[1], 64, generator=gen).to(BF16)
    cond = inp["img"][..., 64:]
    kw = {k: v for k, v in inp.items() if k not in ("img", "timesteps")}
    fn = _sampler(8)
    batched = fn(x.cuda(), model.forward, _cuda(dict(kw, cond=cond)))[-1].float().cpu()
    errs = []
    for b in range(3):
        solo = fn(x[b:b + 1].cuda(), model.forward, _cuda(dict(_pick(kw, b), cond=cond[b:b + 1])))[-1].float().cpu()
        errs.append(rel_l2(batched[b:b + 1], solo))
    _record("small_b3_vs_b1_final_latent_rel_l2", errs=errs)
    assert max(errs) < 1e-2, errs


def test_fullsize_cfgB_b2_matches_solo():
    import bench
    import visualcloze_b200.model as M
    P = M.flux_dev_fill_params()
    with torch.device("cuda"):
        model = M.FluxLoraWrapper(lora_rank=256, params=P)
    model.init_synthetic(0)
    xs, kws = [], []
    for seed in (1234, 99):
        x, kw, Li, Lt = bench.make_inputs("B", seed)
        xs.append(x)
        kws.append(kw)
    kw2 = {k: torch.cat([kws[0][k], kws[1][k]]) for k in kws[0]}
    kw2["guidance"] = torch.tensor([30.0, 3.5]).to(BF16)
    fn = _sampler(6)
    batched = fn(torch.cat(xs).cuda(), model.forward, _cuda(kw2))[-1].float().cpu()
    errs = []
    for b in range(2):
        solo = fn(xs[b].cuda(), model.forward, _cuda({k: v[b:b + 1] for k, v in kw2.items()}))[-1].float().cpu()
        errs.append(rel_l2(batched[b:b + 1], solo))
    _record("fullsize_cfgB_b2_vs_b1_final_latent_rel_l2_5evals", errs=errs)
    del model
    torch.cuda.empty_cache()
    assert max(errs) < 1e-2, errs


# ------------------------------------------------------------------------------------------------
# per-sample first-block cache
# ------------------------------------------------------------------------------------------------
SCALES = [[0.0, 0.003, 1.0, 0.01, 0.3, 0.001, 3.0, 0.03],
          [0.0, 1.0, 0.002, 0.5, 0.005, 2.0, 0.02, 0.001],
          [0.0, 0.02, 0.02, 2.0, 0.001, 0.001, 0.1, 1.0]]


def _spread_imgs(img, scales, seed):
    gen = torch.Generator().manual_seed(seed)
    return [(img.float() + s * torch.randn(img.shape, generator=gen)).to(BF16) for s in scales]


def _run_evals(model, inp, imgs):
    """one prepare for len(imgs) evaluations; -> outputs, per-evaluation per-sample stats"""
    eng = _prepare(model, _cuda(inp), len(imgs))
    outs, stats = [], []
    for k, img in enumerate(imgs):
        outs.append(eng.forward(k, img.cuda()).clone())
        stats.append(eng.sample_cache_stats())
    return outs, stats


def _skips(stats, b):
    seq, prev = [], 0
    for st in stats:
        seq.append(st[b]["skipped"] > prev)
        prev = st[b]["skipped"]
    return seq


@pytest.mark.parametrize("mode", ["merged_bf16", "unmerged", "fp8"])
def test_per_sample_equals_per_batch_at_b1(mode):
    g = _load("flux_small_b1.pt")
    kw = dict(merged_bf16={}, unmerged=dict(lora_mode="unmerged"), fp8=dict(precision="fp8"))[mode]
    model = _build(g["cfg"], g["param_seed"], **kw)
    inp = g["inputs"]
    imgs = _spread_imgs(inp["img"], SCALES[0], 11)
    model.enable_first_block_cache(1e-30)
    _, probe = _run_evals(model, inp, imgs)
    ds = sorted(st[0]["last_diff"] for st in probe[1:])
    checked = []
    for t in [math.sqrt(a * b) for a, b in zip(ds, ds[1:]) if b > 1.5 * a]:
        model.enable_first_block_cache(t)
        o1, s1 = _run_evals(model, inp, imgs)
        c1 = model.cache_stats()
        model.enable_first_block_cache(t, per_sample=True)
        o2, s2 = _run_evals(model, inp, imgs)
        c2 = model.cache_stats()
        assert s1 == s2 and c1 == c2, (t, s1, s2)
        for a, b in zip(o1, o2):
            assert torch.equal(a, b), t
        checked.append((t, c1["skipped"]))
    print(f"[batch] {mode}: per-sample == per-batch bitwise at B = 1, (threshold, skipped): {checked}")
    assert any(0 < n < len(imgs) - 1 for _, n in checked), checked


def test_per_sample_decisions_at_b3_equal_solo_runs():
    g = _load("flux_small_b1.pt")
    model = _build(g["cfg"], g["param_seed"])
    inp3 = _batch_inputs(g["inputs"], 3)
    imgs_b = [_spread_imgs(inp3["img"][b:b + 1], SCALES[b], 20 + b) for b in range(3)]
    imgs = [torch.cat([imgs_b[b][k] for b in range(3)]) for k in range(len(SCALES[0]))]
    model.enable_first_block_cache(1e-30, per_sample=True)
    _, probe = _run_evals(model, inp3, imgs)
    solo_probe = [_run_evals(model, _pick(inp3, b), imgs_b[b])[1] for b in range(3)]
    diffs = sorted({st[b]["last_diff"] for st in probe[1:] for b in range(3)} |
                   {st[0]["last_diff"] for sp in solo_probe for st in sp[1:]})
    checked = []
    for t in [math.sqrt(a * b) for a, b in zip(diffs, diffs[1:]) if b > 1.25 * a]:
        if any(abs(d - t) < 0.1 * t for d in diffs):
            continue
        model.enable_first_block_cache(t, per_sample=True)
        outs, stats = _run_evals(model, inp3, imgs)
        seqs = []
        for b in range(3):
            solo_out, solo_stats = _run_evals(model, _pick(inp3, b), imgs_b[b])
            assert _skips(stats, b) == _skips(solo_stats, 0), (t, b, _skips(stats, b), _skips(solo_stats, 0))
            for k in range(len(imgs)):
                assert rel_l2(outs[k][b:b + 1].float(), solo_out[k].float()) < 2e-2, (t, b, k)
            seqs.append(sum(_skips(stats, b)))
        checked.append((t, seqs))
    print(f"[batch] per-sample decisions at B = 3 equal solo, (threshold, skipped per sample): {checked}")
    assert any(len(set(s)) > 1 for _, s in checked), checked      # samples decided differently in one solve


def test_per_sample_repeated_evaluation_skips_every_sample_bitwise():
    g = _load("flux_small_b1.pt")
    model = _build(g["cfg"], g["param_seed"])
    model.enable_first_block_cache(1e-3, per_sample=True)
    inp = _cuda(_batch_inputs(g["inputs"], 3))
    eng = _prepare(model, inp, 1)
    out1 = eng.forward(0, inp["img"]).clone()
    out2 = eng.forward(0, inp["img"])
    st = eng.sample_cache_stats()
    assert all((s["computed"], s["skipped"], s["last_diff"]) == (1, 1, 0.0) for s in st), st
    assert eng.cache_stats()["skipped"] == 1
    assert torch.equal(out1, out2)


def test_per_sample_padding_is_excluded():
    g = _load("flux_small_b2r.pt")
    inp = _cuda(g["inputs"])
    pad = ~inp["img_mask"].bool()
    assert pad.any()
    gen = torch.Generator(device="cuda").manual_seed(3)
    img_b = (inp["img"].float() + 0.05 * torch.randn(inp["img"].shape, generator=gen, device="cuda")).to(BF16)

    def garbage(x):
        return torch.where(pad[..., None], (300.0 * torch.randn(x.shape, generator=gen, device="cuda")).to(BF16), x)

    for threshold in (1e-6, 1e6):
        model = _build(g["cfg"], g["param_seed"])
        model.enable_first_block_cache(threshold, per_sample=True)
        runs = []
        for a, b in ((inp["img"], img_b), (garbage(inp["img"]), garbage(img_b))):
            eng = _prepare(model, inp, 2)
            o0 = eng.forward(0, a).clone()
            o1 = eng.forward(1, b).clone()
            runs.append((o0, o1, eng.sample_cache_stats()))
        (a0, a1, sa), (b0, b1, sb) = runs
        assert sa == sb, (sa, sb)
        assert all(s["skipped"] == (1 if threshold > 1 else 0) and 0 < s["last_diff"] < math.inf for s in sa), sa
        valid = inp["img_mask"].bool()
        assert torch.equal(a0[valid], b0[valid]) and torch.equal(a1[valid], b1[valid])


def test_per_batch_mode_at_b3_shares_one_decision():
    """per-batch mode at B > 1 through the new entry point (per_sample 0) is the old entry point, bit for bit, and every sample
    reports the batch's counters"""
    from visualcloze_b200._lib import check
    g = _load("flux_small_b1.pt")
    model = _build(g["cfg"], g["param_seed"])
    inp3 = _batch_inputs(g["inputs"], 3)
    imgs = [torch.cat([_spread_imgs(inp3["img"][b:b + 1], SCALES[b], 20 + b)[k] for b in range(3)]) for k in range(len(SCALES[0]))]
    model.enable_first_block_cache(1e-30)
    _, probe = _run_evals(model, inp3, imgs)
    ds = sorted(st[0]["last_diff"] for st in probe[1:])
    eng = model.engine()
    skipped = []
    for t in [math.sqrt(a * b) for a, b in zip(ds, ds[1:])] + [2.0 * ds[-1]]:
        model.enable_first_block_cache(t, per_sample=False)
        o_new, s_new = _run_evals(model, inp3, imgs)
        check(eng.lib.vcb_flux_set_first_block_cache(eng._h, t), "vcb_flux_set_first_block_cache")
        o_old, s_old = _run_evals(model, inp3, imgs)
        assert s_old == s_new and all(st[0] == st[1] == st[2] for st in s_new)
        for a, b in zip(o_old, o_new):
            assert torch.equal(a, b)
        skipped.append(s_new[-1][0]["skipped"])
    assert any(0 < n < len(imgs) - 1 for n in skipped), skipped


# ------------------------------------------------------------------------------------------------
# process_images_batch against solo calls (reduced-size model, stub encoders)
# ------------------------------------------------------------------------------------------------
def _make_pipe():
    from visualcloze_b200 import pipeline as P, vae as V
    g = _load("flux_small_b1.pt")
    model = _build(g["cfg"], g["param_seed"])
    vsmall = dict(ch=64, ch_mult=[1, 2, 2, 2], num_res_blocks=1)
    dec = V.AutoEncoderDecoder(V.AutoEncoderParams(**vsmall), device="cuda").init_synthetic(1)
    return P.VisualClozeModel(None, resolution=64, model=model, ae_decoder=dec, t5=_t5, clip=_clip, encode=_encode)


@pytest.fixture(scope="module")
def rig():
    return _make_pipe()


def _t5(prompts):                     # per prompt, so a batch of prompts gives each row what a solo call gives
    return torch.stack([(0.3 * torch.randn(24, 64, generator=torch.Generator().manual_seed(len(p) * 31 + sum(map(ord, p)))))
                        for p in prompts]).to(BF16).cuda()


def _clip(prompts):
    return torch.stack([torch.randn(32, generator=torch.Generator().manual_seed(sum(map(ord, p)))) for p in prompts]).to(BF16).cuda()


def _encode(x):                       # stands in for AutoencoderKL.encode(x).latent_dist.sample(), one image at a time
    gg = torch.Generator(device="cuda").manual_seed(int(x.shape[-1]) + int(x.float().abs().sum().item() * 7) % 1000)
    return torch.randn(x.shape[0], 16, x.shape[2] // 8, x.shape[3] // 8, generator=gg, device="cuda").to(BF16)


def _psnr(a, b):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return 10 * math.log10(255.0 ** 2 / max(((a - b) ** 2).mean(), 1e-12))


def _grid(gh, gw, seed, size=90):
    from PIL import Image
    rng = np.random.RandomState(seed)
    imgs = [[Image.fromarray(rng.randint(0, 255, (size, size, 3), dtype=np.uint8)) for _ in range(gw)] for _ in range(gh)]
    imgs[-1][-1] = None
    return imgs


def _spy(pipe, seen):
    make = pipe._make_sample_fn

    def wrapped(*a, **k):
        fn = make(*a, **k)

        def spy(x, model, kw):
            seen.append(dict(kw, x=x.clone()))
            return fn(x, model, kw)
        return spy
    pipe._make_sample_fn = wrapped
    return make


_KEYS = ("x", "cond", "img_ids", "txt", "txt_ids", "txt_mask", "y", "img_mask", "guidance")


def _requests():
    from visualcloze_b200.pipeline import GridRequest
    p = ["layout prompt", "task prompt", "The last image of the last row depicts: content"]
    return [GridRequest((2, 3), _grid(2, 3, 0), p, seed=5, cfg=30),
            GridRequest((2, 3), _grid(2, 3, 0), p, seed=6, cfg=30),
            GridRequest((3, 2), _grid(3, 2, 1), ["other layout", "other task", "other content"], seed=7, cfg=3.5),
            GridRequest((1, 2), _grid(1, 2, 2), p, seed=8, cfg=10)]


def _solo(pipe, r, seen, **kw):
    pipe.set_grid_size(*r.grid)
    orig = _spy(pipe, seen)
    try:
        return pipe.process_images([list(row) for row in r.images], list(r.prompts), seed=r.seed, cfg=r.cfg, **kw)
    finally:
        pipe._make_sample_fn = orig


def test_process_images_batch_matches_solo_calls(rig):
    pipe = rig
    reqs = _requests()
    seen = []
    orig = _spy(pipe, seen)
    try:
        out = pipe.process_images_batch(reqs, steps=4, is_upsampling=False, max_batch=4)
    finally:
        pipe._make_sample_fn = orig
    assert [s["x"].shape[0] for s in seen] == [3, 1], "2x3 + 2x3 + 3x2 share a solve (equal Li); 1x2 runs on its own"
    slot = {0: (0, 0), 1: (0, 1), 2: (0, 2), 3: (1, 0)}
    psnrs, bitwise = [], []
    for k, r in enumerate(reqs):
        solo_seen = []
        ref = _solo(pipe, r, solo_seen, steps=4, is_upsampling=False)
        call, b = slot[k]
        for key in _KEYS:
            a, s = seen[call][key][b:b + 1], solo_seen[0][key]
            assert a.shape == s.shape and a.dtype == s.dtype and torch.equal(a.cpu(), s.cpu()), (k, key)
        assert len(out[k]) == len(ref) == 1 and out[k][0].size == ref[0].size
        psnrs.append(_psnr(out[k][0], ref[0]))
        bitwise.append(bool(np.array_equal(np.asarray(out[k][0]), np.asarray(ref[0]))))
    _record("process_images_batch_vs_solo", psnr_db=psnrs, bitwise=bitwise)
    assert min(psnrs) >= 35.0, psnrs


_CHILD = r"""
import json, sys
sys.path.insert(0, sys.argv[1]); sys.path.insert(0, sys.argv[1] + "/tests")
import numpy as np, test_batch_requests_gpu as T
pipe = T._make_pipe()
reqs = T._requests()
out = pipe.process_images_batch(reqs, steps=4, is_upsampling=False, max_batch=4)
eq = [bool(np.array_equal(np.asarray(o[0]), np.asarray(T._solo(pipe, r, [], steps=4, is_upsampling=False)[0]))) for o, r in zip(out, reqs)]
print("BITWISE " + json.dumps(eq))
"""


def test_process_images_batch_bitwise_without_stream_k_recorded():
    """Recorded, not judged: with stream-K off the GEMM tiling depends less on M; whether batched and solo images then agree
    bit for bit."""
    env = dict(os.environ, VCB_STREAMK="0")
    res = subprocess.run([sys.executable, "-c", _CHILD, REPO], env=env, capture_output=True, text=True, timeout=600)
    assert res.returncode == 0, res.stderr[-3000:]
    line = [ln for ln in res.stdout.splitlines() if ln.startswith("BITWISE ")][-1]
    _record("process_images_batch_vs_solo_bitwise_streamk0", bitwise=json.loads(line[8:]))


def test_sdedit_targets_batched_match_solo(rig):
    pipe = rig
    reqs = _requests()[:3:2]                       # two requests, one target each, equal SDEdit size
    seen = []
    orig = _spy(pipe, seen)
    try:
        out = pipe.process_images_batch(reqs, steps=3, upsampling_steps=4, upsampling_noise=0.4, is_upsampling=True, max_batch=4)
    finally:
        pipe._make_sample_fn = orig
    assert [s["x"].shape[0] for s in seen] == [2, 2], "one grid solve (equal Li), one SDEdit solve of both targets"
    sd = seen[-1]
    psnrs = []
    for k, r in enumerate(reqs):
        solo_seen = []
        ref = _solo(pipe, r, solo_seen, steps=3, upsampling_steps=4, upsampling_noise=0.4, is_upsampling=True)
        for key in _KEYS:
            assert torch.equal(sd[key][k:k + 1].cpu(), solo_seen[-1][key].cpu()), (k, key)
        assert len(out[k]) == len(ref) == 1 and out[k][0].size == ref[0].size
        psnrs.append(_psnr(out[k][0], ref[0]))
    _record("sdedit_batch_vs_solo", psnr_db=psnrs)
    assert min(psnrs) >= 35.0, psnrs


def test_process_images_batch_with_cache_decides_per_sample(rig):
    pipe = rig
    pipe.model.enable_first_block_cache(1e6)
    make, seen = pipe._make_sample_fn, []

    def wrapped(*a, **k):
        fn = make(*a, **k)

        def spy(x, model, kw):
            out = fn(x, model, kw)
            seen.append((pipe.model._fbc_per_sample, pipe.model.cache_stats(per_sample=True)))
            return out
        return spy
    pipe._make_sample_fn = wrapped
    try:
        out = pipe.process_images_batch(_requests()[:2], steps=4, is_upsampling=False, max_batch=2)
    finally:
        pipe._make_sample_fn = make
        pipe.model.enable_first_block_cache(None)
    assert len(out) == 2 and len(seen) == 1
    per_sample, st = seen[0]
    assert per_sample and len(st) == 2 and all(s["computed"] == 1 and s["skipped"] == 2 for s in st), seen
    assert pipe.model._fbc_per_sample is False
