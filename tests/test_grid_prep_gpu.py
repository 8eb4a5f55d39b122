"""Grid-cell preparation on the H100, bit for bit: ``vcb_resample_u8`` against ``PIL.Image.resize``; the device-built grid rows
against ``torch.cat([image_transform(c) for c in cells], dim=2)`` of the Pillow path (``_prepare_grid``); the SDEdit model input
built from a decoded tile against Pillow's crop -> resize -> ``image_transform``; and ``process_images`` with upsampling on,
photo-sized inputs, against a second run whose grid and SDEdit preparation are done with Pillow."""
import os

import numpy as np
import pytest
import torch
from PIL import Image

from conftest import GOLDEN
from test_grid_prep_host import SWEEP, grid_cases, make_images

pytestmark = pytest.mark.gpu
BF16 = torch.bfloat16
_PIL = {"lanczos": Image.LANCZOS, "bicubic": Image.BICUBIC}


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    return torch.device("cuda")


def _pm(gh, gw, res, device):
    from visualcloze_b200 import pipeline as P
    pm = object.__new__(P.VisualClozeModel)
    pm.grid_h, pm.grid_w, pm.resolution, pm.device = gh, gw, res, device
    return pm


@pytest.mark.parametrize("filt", ["lanczos", "bicubic"])
@pytest.mark.parametrize("W,H,w,h", SWEEP)
def test_resample_kernel_is_pillow_resize(dev, W, H, w, h, filt):
    from visualcloze_b200 import resample
    a = np.random.default_rng(W * 7 + h).integers(0, 256, (H, W, 3), dtype=np.uint8)
    want = np.asarray(Image.fromarray(a).resize((w, h), _PIL[filt]))
    got = resample.resize(torch.from_numpy(a).to(dev), (w, h), filt)
    assert tuple(got.shape) == (h, w, 3) and np.array_equal(got.cpu().numpy(), want)


def test_resample_reads_a_strided_crop_view(dev):
    """A crop inside the image is a view with the parent's row stride; both passes read it in place."""
    from visualcloze_b200 import resample
    a = np.random.default_rng(5).integers(0, 256, (301, 517, 3), dtype=np.uint8)
    box = (33, 17, 33 + 211, 17 + 257)
    view = resample.crop(torch.from_numpy(a).to(dev), box)
    assert view.stride(0) == 3 * 517
    for filt in ("lanczos", "bicubic"):
        want = np.asarray(Image.fromarray(a).crop(box).resize((97, 140), _PIL[filt]))
        assert np.array_equal(resample.resize(view, (97, 140), filt).cpu().numpy(), want)
    # a box reaching outside the image: a zero-padded copy, as Image.crop pads
    pad = (-20, 290, 60, 320)
    assert np.array_equal(resample.crop(torch.from_numpy(a).to(dev), pad).cpu().numpy(), np.asarray(Image.fromarray(a).crop(pad)))


def test_store_is_image_transform_for_every_value_and_pads_with_minus_one(dev):
    from visualcloze_b200 import ops
    from visualcloze_b200.pipeline import image_transform
    a = np.arange(256 * 3, dtype=np.int64).reshape(16, 16, 3).astype(np.uint8)
    a[..., 1] = a[..., 0][::-1]
    out = torch.full((3, 20, 40), 7.0, device=dev)
    ops.u8_to_model_input(torch.from_numpy(a).to(dev), (-2, -3, 18, 17), out, 5)
    want = image_transform(Image.fromarray(a).crop((-2, -3, 18, 17)))
    assert torch.equal(out[:, :20, 5:25].cpu(), want)
    assert (out[:, :, :5] == 7.0).all() and (out[:, :, 25:] == 7.0).all()
    ops.u8_to_model_input(None, (0, 0, 6, 4), out, 30)                      # a blank cell
    assert (out[:, :4, 30:36] == -1.0).all() and (out[:, 4:, 30:36] == 7.0).all()


def _pil_rows(images, gh, gw, res, device):
    from visualcloze_b200.pipeline import image_transform
    processed, mask, up = _pm(gh, gw, res, device)._prepare_grid(images)
    rows = [torch.cat([image_transform(c) for c in processed[i * gw:(i + 1) * gw]], dim=2).to(device) for i in range(gh)]
    return rows, mask, up


@pytest.mark.parametrize("case", grid_cases(), ids=lambda c: c[0])
def test_device_rows_are_the_pillow_rows(dev, case):
    _, gh, gw, res, sizes = case
    images = make_images(sizes, seed=3)
    want, want_mask, want_up = _pil_rows(images, gh, gw, res, dev)
    got, mask, up = _pm(gh, gw, res, dev)._grid_rows(images)
    assert mask == want_mask and up == want_up and len(got) == gh
    for g, w in zip(got, want):
        assert g.dtype == torch.float32 and g.shape == w.shape and torch.equal(g, w)


def test_device_rows_photo_sized_3x4(dev):
    sizes = [[(4032, 3024)] * 4, [(3024, 4032), (4032, 3024), (3000, 3000), (4032, 2268)], [(4032, 3024), None, None, None]]
    images = make_images(sizes, seed=9)
    want, _, _ = _pil_rows(images, 3, 4, 384, dev)
    got, mask, _ = _pm(3, 4, 384, dev)._grid_rows(images)
    assert mask == [0, 1, 1, 1]
    assert all(torch.equal(g, w) for g, w in zip(got, want))


@pytest.mark.parametrize("H,W,grid_w,target", [(384, 1152, 3, (4032, 3024)), (256, 768, 3, (640, 480)), (96, 192, 2, (97, 131)),
                                               (128, 384, 3, (128, 128))])
def test_sdedit_input_from_a_decoded_tile(dev, H, W, grid_w, target):
    """The SDEdit model input of every target column of a decoded query tile, and the image the noise >= 1 early return gives,
    equal Pillow's crop -> resize (BICUBIC) -> image_transform of the tile."""
    from visualcloze_b200 import ops
    from visualcloze_b200.pipeline import image_transform
    tile = torch.randint(0, 256, (3, H, W), dtype=torch.uint8, device=dev)           # decode_packed's layout
    hwc = tile.permute(1, 2, 0).contiguous()
    query = Image.fromarray(hwc.cpu().numpy())
    pm = _pm(1, grid_w, 384, dev)
    size = target
    if size[0] * size[1] > 1024 * 1024:
        ar = size[0] / size[1]
        nh = int((1024 * 1024 / ar) ** 0.5)
        size = (int(nh * ar), nh)
    size = ((size[0] // 16) * 16, (size[1] // 16) * 16)
    for j in range(grid_w):
        box = (j * W // grid_w, 0, (j + 1) * W // grid_w, H)
        want_img = query.crop(box).resize(size)
        img = pm._sdedit_resize(hwc, box, size)
        assert np.array_equal(img.cpu().numpy(), np.asarray(want_img))
        x = ops.u8_to_model_input(img, (0, 0) + size, torch.empty(3, size[1], size[0], device=dev), 0)
        assert torch.equal(x.cpu(), image_transform(want_img))
        early = pm._upsampling(hwc, box, target, 30, 3, 1.0, None, "x")
        assert early.mode == want_img.mode and early.size == want_img.size and early.tobytes() == want_img.tobytes()
        early = pm.upsampling(query.crop(box), target, 30, 3, 1.0, None, "x")
        assert early.tobytes() == want_img.tobytes()


# ---- process_images end to end ---------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def pipe(dev):
    from oracle import flux_oracle as fo
    import visualcloze_b200.model as M
    from visualcloze_b200 import pipeline as P, vae as V
    g = torch.load(os.path.join(GOLDEN, "flux_small_b1.pt"), weights_only=False)
    cfg = fo.FluxConfig(**g["cfg"])
    fp = M.FluxParams(**{k: v for k, v in g["cfg"].items() if k not in ("lora_rank", "lora_scale")})
    with torch.device("cuda"):
        model = M.FluxLoraWrapper(lora_rank=cfg.lora_rank, params=fp)
    model.load_state_dict({k: v.cuda() for k, v in fo.make_params(cfg, seed=g["param_seed"]).items()}, strict=True)
    dec = V.AutoEncoderDecoder(V.AutoEncoderParams(ch=64, ch_mult=[1, 2, 2, 2], num_res_blocks=1), device="cuda").init_synthetic(1)
    t5 = lambda prompts: (0.3 * torch.randn(len(prompts), 24, 64, generator=torch.Generator().manual_seed(len(prompts[0])))).to(BF16).cuda()
    clip = lambda prompts: torch.randn(len(prompts), 32, generator=torch.Generator().manual_seed(7)).to(BF16).cuda()

    def encode(x):                       # depends on the pixel values, so a changed model input changes the result
        gg = torch.Generator(device="cuda").manual_seed(int(x.shape[-1]) + int(x.float().abs().sum().item() * 7) % 1000)
        return torch.randn(x.shape[0], 16, x.shape[2] // 8, x.shape[3] // 8, generator=gg, device="cuda")
    return P.VisualClozeModel(None, resolution=64, model=model, ae_decoder=dec, t5=t5, clip=clip, encode=encode)


def test_process_images_device_preparation_equals_the_pillow_preparation(pipe, monkeypatch):
    from visualcloze_b200 import resample
    pipe.set_grid_size(2, 3)
    sizes = [[(4032, 3024), (3024, 4032), (2000, 2000)], [(4032, 3024), (1600, 1200), None]]
    prompts = ["layout", "task", "The last image of the last row depicts: a cat"]
    seen = {"device": [], "pillow": []}

    def run(tag):
        enc = pipe._encode_tokens
        monkeypatch.setattr(pipe, "_encode_tokens", lambda x: (seen[tag].append(x.clone()), enc(x))[1])
        out = pipe.process_images(make_images(sizes, seed=1), prompts, seed=5, cfg=30, steps=3, upsampling_steps=2,
                                  upsampling_noise=0.4, is_upsampling=True)
        monkeypatch.undo()
        return out
    out_dev = run("device")

    def pillow_rows(images):
        return _pil_rows(images, pipe.grid_h, pipe.grid_w, pipe.resolution, pipe.device)

    def pillow_sdedit(tile, box, size):
        im = Image.fromarray(tile.cpu().numpy()).crop(box).resize(size)
        return torch.from_numpy(np.array(im)).to(pipe.device)
    monkeypatch.setattr(pipe, "_grid_rows", pillow_rows)
    monkeypatch.setattr(pipe, "_sdedit_resize", pillow_sdedit)
    out_pil = run("pillow")
    assert len(out_dev) == len(out_pil) == 1 and out_dev[0].size == out_pil[0].size == (1168, 880)
    assert len(seen["device"]) == len(seen["pillow"]) == 4          # two grid rows, the SDEdit image and its blank
    for a, b in zip(seen["device"], seen["pillow"]):
        assert a.shape == b.shape and torch.equal(a, b)
    assert out_dev[0].tobytes() == out_pil[0].tobytes()
