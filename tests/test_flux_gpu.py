"""Model-level parity on the H100: Flux.forward and the Euler sampler through the reference-shaped Python API
(visualcloze_b200.model / transport -> libvcb200.so) against the CPU oracle and the reference-generated goldens.

Tolerances (SURVEY.md 8c; reference-vs-reference noise, FA2 vs SDPA and merged vs un-merged LoRA, is ~1e-2):
  block-level / reduced-depth forward   rel-L2 <= 2e-2
  multi-step trajectory, final latent   rel-L2 <= 5e-2
"""
import os

import pytest
import torch

from conftest import GOLDEN, rel_l2

pytestmark = pytest.mark.gpu
BF16 = torch.bfloat16


@pytest.fixture(scope="module")
def vcb():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    import visualcloze_b200.model as m
    import visualcloze_b200.transport as t
    return m, t


def _load(name):
    return torch.load(os.path.join(GOLDEN, name), weights_only=False)


def _build(m, cfg_dict, seed):
    from oracle import flux_oracle as fo
    cfg = fo.FluxConfig(**cfg_dict)
    params = fo.make_params(cfg, seed=seed)
    fp = m.FluxParams(**{k: v for k, v in cfg_dict.items() if k not in ("lora_rank", "lora_scale")})
    with torch.device("cuda"):
        model = m.FluxLoraWrapper(lora_rank=cfg.lora_rank, params=fp)
    missing = model.load_state_dict({k: v.cuda() for k, v in params.items()}, strict=True)
    assert not missing.missing_keys and not missing.unexpected_keys
    return cfg, params, model


def _cuda(d):
    return {k: (v.cuda() if torch.is_tensor(v) else v) for k, v in d.items()}


@pytest.mark.parametrize("tag", ["b1", "b2r"])
def test_forward_small_vs_oracle_and_reference_golden(vcb, tag):
    m, _ = vcb
    from oracle import flux_oracle as fo
    g = _load(f"flux_small_{tag}.pt")
    cfg, params, model = _build(m, g["cfg"], g["param_seed"])
    inp = g["inputs"]
    keep = {k: v.clone() for k, v in inp.items()}
    out = model(**_cuda(inp)).cpu()
    assert out.dtype == BF16 and out.shape == g["out_cpu_bf16"].shape
    assert all(torch.equal(inp[k], keep[k]) for k in inp), "inputs must not be mutated"
    ref = fo.flux_forward(params, cfg, **inp, mode="cuda_bf16")
    mask = inp["img_mask"].bool()
    # padded img rows (batch > 1) are don't-care in the reference as well: compare valid tokens
    e_or = rel_l2(out[mask], ref[mask])
    e_gold = rel_l2(out[mask], g["out_cpu_bf16"][mask])
    assert e_or < 2e-2, f"vs oracle {e_or:.3e}"
    assert e_gold < 2.5e-2, f"vs reference golden {e_gold:.3e}"


def test_forward_errors_match_reference(vcb):
    m, _ = vcb
    g = _load("flux_small_b1.pt")
    _, _, model = _build(m, g["cfg"], g["param_seed"])
    inp = _cuda(g["inputs"])
    with pytest.raises(ValueError, match="3 dimensions"):
        model(**dict(inp, img=inp["img"][0]))
    with pytest.raises(ValueError, match="guidance"):
        model(**dict(inp, guidance=None))


def test_forward_full_width_reduced_depth(vcb):
    """FLUX geometry (hidden 3072, 24 heads, mlp 12288, ctx 4096, LoRA on every Linear) at depth 1+1."""
    m, _ = vcb
    from oracle import flux_oracle as fo
    cfg_dict = dict(in_channels=384, out_channels=64, vec_in_dim=768, context_in_dim=4096, hidden_size=3072, mlp_ratio=4.0,
                    num_heads=24, depth=1, depth_single_blocks=1, axes_dim=[16, 56, 56], theta=10_000, qkv_bias=True,
                    guidance_embed=True, lora_rank=32)
    cfg, params, model = _build(m, cfg_dict, seed=21)
    g = torch.Generator().manual_seed(5)
    B, rows, Lt = 1, [(6, 18), (6, 18)], 96
    ids = []
    for j, (h, w) in enumerate(rows):
        t = torch.zeros(h, w, 3)
        t[..., 0] = j + 1
        t[..., 1] += torch.arange(h)[:, None]
        t[..., 2] += torch.arange(w)[None, :]
        ids.append(t.reshape(-1, 3))
    ids = torch.cat(ids)[None]
    Li = ids.shape[1]
    inp = dict(img=torch.randn(B, Li, 384, generator=g).to(BF16), img_ids=ids,
               txt=(0.1 * torch.randn(B, Lt, 4096, generator=g)).to(BF16), txt_ids=torch.zeros(B, Lt, 3),
               timesteps=torch.tensor([0.63]), y=torch.randn(B, 768, generator=g).to(BF16),
               txt_mask=torch.ones(B, Lt, dtype=torch.int32), img_mask=torch.ones(B, Li, dtype=torch.int32),
               guidance=torch.full((B,), 30.0, dtype=BF16))
    out = model(**_cuda(inp)).cpu()
    ref = fo.flux_forward(params, cfg, **inp, mode="cuda_bf16")
    e = rel_l2(out, ref)
    assert e < 2e-2, f"rel_l2 {e:.3e}"


@pytest.mark.parametrize("tag", ["shift4", "sdedit5"])
def test_sampler_trajectory(vcb, tag):
    """Sampler.sample_ode(...)(x, model.forward, kwargs): native fast path vs oracle loop vs reference golden."""
    m, t = vcb
    from oracle import flux_oracle as fo
    from oracle import sampler_oracle as so
    gs = _load("sampler.pt")[tag]
    gf = _load("flux_small_b1.pt")
    cfg, params, model = _build(m, gf["cfg"], gf["param_seed"])
    kw = dict(gs["kwargs"])
    sampler = t.Sampler(t.create_transport("Linear", "velocity", do_shift=True))
    fn = sampler.sample_ode(sampling_method="euler", atol=1e-6, rtol=1e-3, reverse=False, **kw)
    mk = dict(_cuda(gs["inputs"]), cond=gs["cond"].cuda())
    traj = fn(gs["x"].cuda(), model.forward, mk).cpu()
    assert "cond" in mk
    assert traj.shape == gs["traj"].shape and traj.dtype == BF16
    assert torch.equal(traj[0], gs["x"])

    def model_fn(x, timesteps, **k):
        return fo.flux_forward(params, cfg, img=x, timesteps=timesteps, **k, mode="cuda_bf16")

    ref = so.sample_ode(gs["x"], model_fn, dict(gs["inputs"], cond=gs["cond"]), num_steps=kw["num_steps"],
                        do_shift=kw["do_shift"], time_shifting_factor=kw["time_shifting_factor"], strength=kw.get("strength"))
    e_or, e_gold = rel_l2(traj[-1], ref[-1]), rel_l2(traj[-1], gs["traj"][-1])
    assert e_or < 5e-2, f"vs oracle {e_or:.3e}"
    assert e_gold < 5e-2, f"vs reference golden {e_gold:.3e}"
    # first step is a single evaluation: tighter
    assert rel_l2(traj[1], ref[1]) < 1e-2

    # generic path (foreign callable) must give the same trajectory as the fast path
    calls = []

    def foreign(x, timesteps, **k):
        calls.append(float(timesteps[0]))
        return model(x, timesteps=timesteps, **k)

    traj2 = fn(gs["x"].cuda(), foreign, mk).cpu()
    assert len(calls) == kw["num_steps"] - 1
    assert torch.allclose(torch.tensor(calls), gs["flux_t"].flatten(), atol=1e-6)
    assert rel_l2(traj2[-1], traj[-1]) < 1e-2


def test_lora_scale_repacks(vcb):
    m, _ = vcb
    g = _load("flux_small_b1.pt")
    _, _, model = _build(m, g["cfg"], g["param_seed"])
    inp = _cuda(g["inputs"])
    a = model(**inp)
    model.set_lora_scale(0.0)
    b = model(**inp)
    model.set_lora_scale(1.0)
    c = model(**inp)
    assert torch.equal(a, c)
    assert rel_l2(a.cpu(), b.cpu()) > 1e-3, "LoRA branch must contribute"


def test_pipeline_process_images_end_to_end(vcb):
    """VisualClozeModel.process_images (visualcloze.py:247-467) with injected text / VAE-encode stubs: query-row crop of the
    right size, seed-deterministic, equal to composing sampler + decoder by hand; SDEdit upsampling path runs."""
    m, t = vcb
    from PIL import Image
    from visualcloze_b200 import pipeline as P, vae as V
    g = _load("flux_small_b1.pt")
    _, _, model = _build(m, g["cfg"], g["param_seed"])
    dec = V.AutoEncoderDecoder(V.AutoEncoderParams(ch=64, ch_mult=[1, 2, 2, 2], num_res_blocks=1), device="cuda").init_synthetic(1)
    t5 = lambda prompts: (0.3 * torch.randn(len(prompts), 24, 64, generator=torch.Generator().manual_seed(len(prompts[0])))).to(BF16).cuda()
    clip = lambda prompts: torch.randn(len(prompts), 32, generator=torch.Generator().manual_seed(7)).to(BF16).cuda()

    def encode(x):
        gg = torch.Generator(device="cuda").manual_seed(int(x.shape[-1]))
        return torch.randn(x.shape[0], 16, x.shape[2] // 8, x.shape[3] // 8, generator=gg, device="cuda")

    pipe = P.VisualClozeModel(None, resolution=64, model=model, ae_decoder=dec, t5=t5, clip=clip, encode=encode)
    pipe.set_grid_size(2, 3)
    mk = lambda: [[Image.new("RGB", (90, 90), (40 * i, 60 * j, 128)) for j in range(3)] for i in range(2)]
    imgs = mk(); imgs[1][2] = None
    out = pipe.process_images(imgs, ["layout", "task", "content"], seed=5, cfg=30, steps=4, is_upsampling=False)
    assert len(out) == 1 and out[0].size == (64, 64)
    imgs = mk(); imgs[1][2] = None
    out2 = pipe.process_images(imgs, ["layout", "task", "content"], seed=5, cfg=30, steps=4, is_upsampling=False)
    assert list(out[0].getdata()) == list(out2[0].getdata()), "same seed -> same image"
    imgs = mk(); imgs[1][2] = None
    out3 = pipe.process_images(imgs, ["layout", "task", "content"], seed=6, cfg=30, steps=4, is_upsampling=False)
    assert list(out[0].getdata()) != list(out3[0].getdata())
    imgs = mk(); imgs[1][2] = None
    up = pipe.process_images(imgs, ["layout", "task", "The last image of the last row depicts: a cat"], seed=5, cfg=30, steps=4,
                             upsampling_steps=3, upsampling_noise=0.4, is_upsampling=True)
    assert len(up) == 1 and up[0].size == (80, 80)          # resized to the input cell's size, multiples of 16
    # same pipeline with the library's own VAE encoder for the condition rows (SURVEY.md 8f-1) instead of an injected one
    enc = V.AutoEncoderEncoder(V.AutoEncoderParams(ch=64, ch_mult=[1, 2, 2, 2], num_res_blocks=1), device="cuda").init_synthetic(2)
    pipe2 = P.VisualClozeModel(None, resolution=64, model=model, ae_decoder=dec, ae_encoder=enc, t5=t5, clip=clip)
    pipe2.set_grid_size(2, 3)
    imgs = mk(); imgs[1][2] = None
    out4 = pipe2.process_images(imgs, ["layout", "task", "content"], seed=5, cfg=30, steps=4, is_upsampling=False)
    assert len(out4) == 1 and out4[0].size == (64, 64)
