"""VAE decoder parity on the H100 (autoencoder.py:183-259 via libvcb200) against the CPU oracle / reference golden.
bf16 activations vs the reference's fp32 golden: rel-L2 <= 3e-2 (the decoder is ~25 bf16 conv layers deep);
decoded-image PSNR vs the oracle run with the same bf16 weights >= 35 dB (SURVEY.md 8c)."""
import math
import os

import pytest
import torch

from conftest import GOLDEN, rel_l2

pytestmark = pytest.mark.gpu
BF16 = torch.bfloat16


@pytest.fixture(scope="module")
def mods():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    from visualcloze_b200 import _lib, vae
    return _lib, vae


@pytest.mark.parametrize("shape", [(1, 20, 36, 64, 128), (2, 9, 17, 128, 256), (1, 33, 40, 256, 8), (1, 16, 16, 512, 512)])
@pytest.mark.parametrize("with_res", [False, True])
def test_conv3x3_implicit_gemm(mods, shape, with_res):
    """3x3 / stride 1 / zero pad 1 conv as implicit GEMM with TMA zero-fill padding vs F.conv2d."""
    _lib, _ = mods
    n, H, W, ci, co = shape
    g = torch.Generator().manual_seed(ci + co)
    x = torch.randn(n, ci, H, W, generator=g).to(BF16)
    w = (torch.randn(co, ci, 3, 3, generator=g) / math.sqrt(9 * ci)).to(BF16)
    b = torch.randn(co, generator=g) * 0.1
    res = torch.randn(n, co, H, W, generator=g).to(BF16) if with_res else None
    xg = x.permute(0, 2, 3, 1).contiguous().cuda()
    wg = w.permute(0, 2, 3, 1).reshape(co, 9 * ci).contiguous().cuda()
    rg = None if res is None else res.permute(0, 2, 3, 1).contiguous().cuda()
    out = torch.zeros(n, H, W, co, dtype=BF16, device="cuda")
    _lib.check(_lib.lib().vcb_conv3x3_nhwc(xg.data_ptr(), wg.data_ptr(), b.cuda().data_ptr(), None if rg is None else rg.data_ptr(),
                                           out.data_ptr(), n, H, W, ci, co, 1, None), "conv")
    torch.cuda.synchronize()
    ref = torch.nn.functional.conv2d(x.float(), w.float(), b, padding=1).to(BF16)
    if res is not None:
        ref = res + ref
    got = out.permute(0, 3, 1, 2).cpu()
    assert rel_l2(got, ref) < 4e-3, f"rel_l2={rel_l2(got, ref):.3e}"


def test_decode_small_vs_reference_golden(mods):
    _, vae = mods
    from oracle import vae_oracle as vo
    g = torch.load(os.path.join(GOLDEN, "vae_small.pt"), weights_only=False)
    cfg = vo.VaeConfig(**g["cfg"])
    p = vo.make_decoder_params(cfg, seed=g["param_seed"], dtype=torch.float32)
    dec = vae.AutoEncoderDecoder(vae.AutoEncoderParams(**g["cfg"]), device="cuda")
    missing = dec.load_state_dict({k: v.cuda() for k, v in p.items()}, strict=True)
    assert not missing.missing_keys
    out = dec.decode(g["z"].to(BF16).cuda()).float().cpu()
    assert out.shape == g["out_fp32"].shape
    e = rel_l2(out, g["out_fp32"])
    assert e < 3e-2, f"rel_l2 vs fp32 reference {e:.3e}"


def test_decode_flux_geometry_vs_oracle_and_uint8_path(mods):
    """Full FLUX VAE widths (128/256/512/512, 2 res blocks) on a small latent; oracle runs the same bf16 weights."""
    _, vae = mods
    from oracle import vae_oracle as vo
    cfg = vo.VaeConfig()
    p = vo.make_decoder_params(cfg, seed=11, dtype=BF16)
    dec = vae.AutoEncoderDecoder(device="cuda")
    dec.load_state_dict({k: v.cuda() for k, v in p.items()}, strict=True)
    gen = torch.Generator().manual_seed(2)
    h, w = 4, 6                                             # tokens -> latent 8 x 12 -> image 64 x 96
    tok = torch.randn(1, h * w, 64, generator=gen).to(BF16)
    z = tok.reshape(1, h, w, 16, 2, 2).permute(0, 3, 1, 4, 2, 5).reshape(1, 16, 2 * h, 2 * w)
    out = dec.decode(z.cuda()).float().cpu()
    ref = vo.decode({k: v.float() for k, v in p.items()}, cfg, z.float())
    e = rel_l2(out, ref)
    mse = ((out - ref).clamp(-2, 2) ** 2).mean().item()
    psnr = 10 * math.log10(4.0 / max(mse, 1e-12))           # images span [-1, 1]
    assert e < 3e-2 and psnr > 35, f"rel_l2={e:.3e} psnr={psnr:.1f} dB"
    img = dec.decode_packed(tok.cuda(), h, w).cpu()
    assert img.dtype == torch.uint8 and img.shape == (1, 3, 16 * h, 16 * w)
    exp = (((out.to(BF16) + 1.0) / 2.0).clamp(0, 1).float() * 255).to(torch.uint8)
    assert (img.int() - exp.int()).abs().max() <= 1


# ------------------------------------------------------------------------------------------------
# encoder ("next" row (f)-1): stride-2 conv through TMA element strides, Encoder, sampling + packing
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("shape", [(1, 16, 32, 64, 64), (2, 18, 10, 128, 128), (1, 48, 40, 256, 256)])
def test_conv3x3_stride2_downsample(mods, shape):
    """Downsample (autoencoder.py:85-95): pad (0,1,0,1) then 3x3 stride-2 conv == implicit GEMM with elementStrides 2."""
    _lib, _ = mods
    n, H, W, ci, co = shape
    g = torch.Generator().manual_seed(H * W)
    x = torch.randn(n, ci, H, W, generator=g).to(BF16)
    w = (torch.randn(co, ci, 3, 3, generator=g) / math.sqrt(9 * ci)).to(BF16)
    b = torch.randn(co, generator=g) * 0.1
    xg = x.permute(0, 2, 3, 1).contiguous().cuda()
    wg = w.permute(0, 2, 3, 1).reshape(co, 9 * ci).contiguous().cuda()
    out = torch.zeros(n, H // 2, W // 2, co, dtype=BF16, device="cuda")
    _lib.check(_lib.lib().vcb_conv3x3_nhwc(xg.data_ptr(), wg.data_ptr(), b.cuda().data_ptr(), None, out.data_ptr(), n, H, W, ci, co, 2, None), "conv s2")
    torch.cuda.synchronize()
    ref = torch.nn.functional.conv2d(torch.nn.functional.pad(x.float(), (0, 1, 0, 1)), w.float(), b, stride=2).to(BF16)
    got = out.permute(0, 3, 1, 2).cpu()
    assert got.shape == ref.shape and rel_l2(got, ref) < 4e-3, f"rel_l2={rel_l2(got, ref):.3e}"


def test_encode_small_vs_reference_golden(mods):
    _, vae = mods
    from oracle import vae_oracle as vo
    g = torch.load(os.path.join(GOLDEN, "vae_small.pt"), weights_only=False)
    cfg = vo.VaeConfig(**g["cfg"])
    p = vo.make_encoder_params(cfg, seed=g["enc_param_seed"], dtype=torch.float32)
    enc = vae.AutoEncoderEncoder(vae.AutoEncoderParams(**g["cfg"]), device="cuda")
    assert not enc.load_state_dict({k: v.cuda() for k, v in p.items()}, strict=True).missing_keys
    tok, mom = enc.encode_packed(g["img"].cuda(), None, return_moments=True)
    e = rel_l2(mom.cpu(), g["moments_fp32"])
    assert mom.shape == g["moments_fp32"].shape and e < 3e-2, f"moments rel_l2 vs fp32 reference {e:.3e}"
    # distribution mode: tokens == patchify(scale * (mean - shift))
    mean = g["moments_fp32"][:, :16]
    z = cfg.scale_factor * (mean - cfg.shift_factor)
    ref_tok = z.reshape(1, 16, 8, 2, 12, 2).permute(0, 2, 4, 1, 3, 5).reshape(1, 96, 64)
    assert rel_l2(tok.float().cpu(), ref_tok) < 3e-2


def test_encode_flux_geometry_sampling_and_packing(mods):
    _, vae = mods
    from oracle import vae_oracle as vo
    cfg = vo.VaeConfig()
    p = vo.make_encoder_params(cfg, seed=12, dtype=BF16)
    enc = vae.AutoEncoderEncoder(device="cuda")
    enc.load_state_dict({k: v.cuda() for k, v in p.items()}, strict=True)
    gen = torch.Generator().manual_seed(3)
    img = torch.randn(1, 3, 64, 96, generator=gen).clamp(-1, 1)
    noise = torch.randn(1, 16, 8, 12, generator=gen)
    tok, mom = enc.encode_packed(img.cuda(), noise.cuda(), return_moments=True)
    pf = {k: v.float() for k, v in p.items()}
    ref_mom = vo.encode_moments(pf, cfg, img.to(BF16).float())
    e = rel_l2(mom.cpu(), ref_mom)
    assert e < 3e-2, f"moments rel_l2 {e:.3e}"
    # sampling + scaling + packing applied to the kernel's own moments (isolates the elementwise tail): bf16-exact up to 1 ulp
    mean, logvar = mom.cpu()[:, :16], mom.cpu()[:, 16:]
    z = cfg.scale_factor * (mean + torch.exp(0.5 * logvar) * noise - cfg.shift_factor)
    ref_tok = z.reshape(1, 16, 4, 2, 6, 2).permute(0, 2, 4, 1, 3, 5).reshape(1, 24, 64)
    assert rel_l2(tok.float().cpu(), ref_tok) < 8e-3
