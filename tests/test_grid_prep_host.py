"""CPU checks of the grid-cell preparation: Pillow's fixed-point resampling tables (``visualcloze_b200.resample``) driving an
integer numpy restatement of the two passes equal ``PIL.Image.resize`` bit for bit; the size plan (``pipeline.grid_plan``)
executed with Pillow reproduces the reference's ``_prepare_grid`` cells; the fp32 form the store kernel uses equals
``image_transform``; and the C ABI of ``vcb_resample_u8`` / ``vcb_u8_to_model_input`` (signatures and refusals)."""
import ctypes as C
import os
import re

import numpy as np
import pytest
import torch
from PIL import Image

from conftest import REPO

_PIL = {"lanczos": Image.LANCZOS, "bicubic": Image.BICUBIC}

# (in w, in h, out w, out h): 12x downscale, 4x upscale, 1-pixel outputs, odd and prime sizes, one axis unchanged, same size
SWEEP = [(4032, 3024, 432, 320), (7, 5, 28, 20), (1000, 999, 1, 1), (97, 131, 384, 383), (640, 480, 640, 240),
         (513, 257, 129, 257), (300, 200, 300, 200), (1024, 1024, 1182, 886), (101, 53, 37, 211), (31, 17, 1, 5), (1, 1, 3, 2)]


def _pass(a: np.ndarray, n_out: int, filt: str, axis: int) -> np.ndarray:
    """One pass of the 8-bit resampler along ``axis`` (1 = x, 0 = y) of an [h, w, 3] uint8 image, in integers."""
    from visualcloze_b200 import resample
    a = np.moveaxis(a, axis, 0).astype(np.int64)
    bounds, coeffs = resample.coeffs_8bpc(a.shape[0], n_out, filt)
    out = np.empty((n_out,) + a.shape[1:], np.uint8)
    for i in range(n_out):
        xmin, n = bounds[i]
        s = (1 << 21) + np.tensordot(coeffs[i, :n].astype(np.int64), a[xmin:xmin + n], axes=(0, 0))
        out[i] = np.clip(s >> 22, 0, 255)
    return np.moveaxis(out, 0, axis)


def np_resize(a: np.ndarray, size, filt: str) -> np.ndarray:
    w, h = size
    if a.shape[1] != w:
        a = _pass(a, w, filt, 1)
    if a.shape[0] != h:
        a = _pass(a, h, filt, 0)
    return a


@pytest.mark.parametrize("filt", ["lanczos", "bicubic"])
@pytest.mark.parametrize("W,H,w,h", SWEEP)
def test_tables_drive_a_bit_exact_pillow_resize(W, H, w, h, filt):
    a = np.random.default_rng(W * 7 + h).integers(0, 256, (H, W, 3), dtype=np.uint8)
    want = np.asarray(Image.fromarray(a).resize((w, h), _PIL[filt]))
    assert np.array_equal(np_resize(a, (w, h), filt), want)


def test_tables_shape_and_windows():
    from visualcloze_b200 import resample
    for n_in, n_out, filt in ((4032, 432, "lanczos"), (7, 28, "bicubic"), (1000, 1, "lanczos"), (5, 5, "bicubic")):
        bounds, coeffs = resample.coeffs_8bpc(n_in, n_out, filt)
        assert bounds.dtype == coeffs.dtype == np.int32 and bounds.shape == (n_out, 2) and coeffs.shape[0] == n_out
        support = {"lanczos": 3.0, "bicubic": 2.0}[filt] * max(n_in / n_out, 1.0)
        assert coeffs.shape[1] == 2 * int(np.ceil(support)) + 1
        xmin, n = bounds[:, 0], bounds[:, 1]
        assert (xmin >= 0).all() and (n >= 1).all() and (xmin + n <= n_in).all() and (n <= coeffs.shape[1]).all()
        for i in range(n_out):                     # normalised to 1 in 22-bit fixed point (up to the per-tap rounding)
            assert abs(int(coeffs[i].sum()) - (1 << 22)) <= coeffs.shape[1]
            assert not coeffs[i, n[i]:].any()
    with pytest.raises(ValueError):
        resample.coeffs_8bpc(0, 4, "bicubic")


# ---- the size plan -----------------------------------------------------------------------------------------------------------
def _reference_prepare_grid(images, grid_h, grid_w, resolution):
    """visualcloze.py:300-360 as the pipeline ran it with Pillow alone: every resize and crop done on the images."""
    from visualcloze_b200.pipeline import resize_with_aspect_ratio

    def center_crop(image, target_size):
        w, h = image.size
        nw, nh = target_size
        left, top = (w - nw) // 2, (h - nh) // 2
        return image.crop((left, top, left + nw, top + nh))
    processed, mask_position = [], []
    target_size = upsampling_size = None
    for i in range(grid_h):
        reference_size = None
        for j in range(grid_w):
            if images[i][j] is not None:
                if i == grid_h - 1 and upsampling_size is None:
                    upsampling_size = images[i][j].size
                reference_size = resize_with_aspect_ratio(images[i][j], resolution).size
                if i == grid_h - 1 and target_size is None:
                    target_size = reference_size
                break
        for j in range(grid_w):
            if images[i][j] is not None:
                t = resize_with_aspect_ratio(images[i][j], resolution)
                if t.width <= t.height:
                    t = t.resize((reference_size[0], int(reference_size[0] / t.width * t.height)))
                else:
                    t = t.resize((int(reference_size[1] / t.height * t.width), reference_size[1]))
                processed.append(center_crop(t, reference_size))
                if i == grid_h - 1:
                    mask_position.append(0)
            else:
                if i != grid_h - 1:
                    raise ValueError("Please provide each image in the in-context example.")
                processed.append(Image.new("RGB", reference_size or (resolution, resolution), (0, 0, 0)))
                mask_position.append(1)
    if len(mask_position) > 1 and sum(mask_position) > 1:
        new_w = 384 if target_size is None else target_size[0]
        for k, im in enumerate(processed):
            new_h = int(im.height * (new_w / im.width))
            new_w, new_h = int(new_w / 16) * 16, int(new_h / 16) * 16
            processed[k] = im.resize((new_w, new_h))
    return processed, mask_position, upsampling_size


def _img(w, h, seed):
    return Image.fromarray(np.random.default_rng(seed).integers(0, 256, (h, w, 3), dtype=np.uint8))


def grid_cases():
    """(name, grid_h, grid_w, resolution, sizes) -- sizes[i][j] = (w, h) or None; shared with the GPU tests."""
    return [
        ("2x3_one_target", 2, 3, 384, [[(640, 480), (500, 500), (480, 640)], [(800, 600), (700, 500), None]]),
        ("3x4_cfgD_mask_0111", 3, 4, 384, [[(640, 480)] * 4, [(512, 512), (600, 400), (400, 600), (512, 512)],
                                          [(1000, 750), None, None, None]]),
        ("crop_padding_mixed_aspect", 2, 3, 256, [[(300, 900), (500, 500), (640, 600)], [(900, 300), (700, 500), None]]),
        ("tiny_inputs", 2, 3, 128, [[(7, 5), (3, 11), (16, 16)], [(9, 9), (5, 2), None]]),
        ("multi_target_crop_padding", 2, 3, 192, [[(300, 900), (500, 500), (250, 251)], [(333, 555), None, None]]),
        ("last_row_all_blank", 2, 2, 96, [[(120, 90), (90, 120)], [None, None]]),
    ]


def make_images(sizes, seed=0):
    return [[None if s is None else _img(s[0], s[1], seed + 31 * i + j) for j, s in enumerate(row)] for i, row in enumerate(sizes)]


@pytest.mark.parametrize("case", grid_cases(), ids=lambda c: c[0])
def test_plan_executed_with_pillow_is_the_reference_prepare_grid(case):
    from visualcloze_b200 import pipeline as P
    _, gh, gw, res, sizes = case
    images = make_images(sizes)
    want, want_mask, want_up = _reference_prepare_grid(images, gh, gw, res)
    pm = object.__new__(P.VisualClozeModel)
    pm.grid_h, pm.grid_w, pm.resolution = gh, gw, res
    got, mask, up = pm._prepare_grid(images)
    assert mask == want_mask and up == want_up and len(got) == len(want)
    for a, b in zip(got, want):
        assert a.mode == b.mode and a.size == b.size and a.tobytes() == b.tobytes()
    cells, mask2, up2 = P.grid_plan(sizes, gh, gw, res)
    assert mask2 == mask and up2 == up and [c.size for c in cells] == [im.size for im in want]


def test_plan_covers_crop_padding_and_never_resamples():
    """The plan is sizes only: the padding case (a crop box reaching outside the resized image) is present, and planning a grid
    of photo-sized inputs does no pixel work."""
    from visualcloze_b200 import pipeline as P
    cells, _, _ = P.grid_plan(grid_cases()[2][4], 2, 3, 256)
    boxes = [op[1] for c in cells for op in c.ops if op[0] == "crop"]
    assert any(l < 0 for l, _, _, _ in boxes) and any(t < 0 for _, t, _, _ in boxes)
    cells, mask, up = P.grid_plan([[(4032, 3024)] * 4] * 2 + [[(4032, 3024), None, None, None]], 3, 4, 384)
    assert mask == [0, 1, 1, 1] and up == (4032, 3024)
    assert cells[0].ops[0] == ("resize", (432, 320), "lanczos") and cells[-1].blank == (432, 320)
    with pytest.raises(ValueError, match="in-context"):
        P.grid_plan([[(10, 10), None], [(10, 10), None]], 2, 2, 64)


def test_store_arithmetic_is_image_transform():
    """The store kernel computes (u / 255 - 0.5) / 0.5 with IEEE fp32 division and subtraction; that is image_transform's
    value for every uint8, while a multiply by the reciprocal is not."""
    from visualcloze_b200.pipeline import image_transform
    u = np.arange(256, dtype=np.uint8)
    want = image_transform(Image.fromarray(np.repeat(u[None, :, None], 3, axis=2))).numpy()[0, 0]
    f = u.astype(np.float32)
    got = (f / np.float32(255) - np.float32(0.5)) / np.float32(0.5)
    assert got.dtype == np.float32 and np.array_equal(got.view(np.int32), want.view(np.int32))
    recip = (f * np.float32(1 / 255) - np.float32(0.5)) / np.float32(0.5)
    assert not np.array_equal(recip.view(np.int32), want.view(np.int32))


# ---- C ABI ----------------------------------------------------------------------------------------------------------------
def test_ctypes_prototypes_match_the_header():
    from visualcloze_b200 import _lib
    header = open(os.path.join(REPO, "include", "vcb200.h")).read()
    assert re.search(r"int vcb_resample_u8\(const void\* in, int64_t in_ld, int32_t in_w, int32_t in_h, int32_t axis, "
                     r"const int32_t\* bounds,\s+const int32_t\* coeffs, int32_t ksize, int32_t out_n, void\* out, "
                     r"int64_t out_ld, void\* stream\);", header)
    assert re.search(r"int vcb_u8_to_model_input\(const void\* in, int64_t in_ld, int32_t in_w, int32_t in_h, int32_t crop_x, "
                     r"int32_t crop_y,\s+int32_t crop_w, int32_t crop_h, float\* out, int64_t out_ld_row, "
                     r"int64_t out_ld_plane, int32_t col0,\s+void\* stream\);", header)
    i32, i64, p = C.c_int32, C.c_int64, C.c_void_p
    assert _lib._SIGNATURES["vcb_resample_u8"] == (C.c_int, [p, i64, i32, i32, i32, p, p, i32, i32, p, i64, p])
    assert _lib._SIGNATURES["vcb_u8_to_model_input"] == (C.c_int, [p, i64, i32, i32, i32, i32, i32, i32, p, i64, i64, i32, p])
    lib = _lib.lib()
    assert lib.vcb_resample_u8.restype is C.c_int and lib.vcb_u8_to_model_input.restype is C.c_int


P1, P2, P3, P4 = (C.c_void_p(v) for v in (256, 512, 768, 1024))
# (in, in_ld, in_w, in_h, axis, bounds, coeffs, ksize, out_n, out, out_ld)
_RESAMPLE_OK = (P1, 30, 10, 4, 0, P2, P3, 5, 6, P4, 18)
_RESAMPLE_BAD = {
    "null in": dict(i=0, v=None), "null bounds": dict(i=5, v=None), "null coeffs": dict(i=6, v=None), "null out": dict(i=9, v=None),
    "axis 2": dict(i=4, v=2), "axis -1": dict(i=4, v=-1), "in_w 0": dict(i=2, v=0), "in_h -3": dict(i=3, v=-3),
    "out_n 0": dict(i=8, v=0), "ksize 0": dict(i=7, v=0), "in_ld < 3 in_w": dict(i=1, v=29), "out_ld < 3 out_w": dict(i=10, v=17),
}


@pytest.mark.parametrize("what", sorted(_RESAMPLE_BAD))
def test_resample_refuses_bad_arguments(what):
    """Argument checks run before any device work, so they are exercised without a GPU."""
    from visualcloze_b200 import _lib
    args = list(_RESAMPLE_OK)
    args[_RESAMPLE_BAD[what]["i"]] = _RESAMPLE_BAD[what]["v"]
    assert _lib.lib().vcb_resample_u8(*args, None) != 0
    assert _lib.lib().vcb_last_error().startswith(b"resample_u8:")


# (in, in_ld, in_w, in_h, crop_x, crop_y, crop_w, crop_h, out, out_ld_row, out_ld_plane, col0)
_STORE_OK = (P1, 30, 10, 4, -1, -1, 8, 6, P2, 20, 120, 12)
_STORE_BAD = {
    "null out": dict(i=8, v=None), "null in": dict(i=0, v=None), "crop_w 0": dict(i=6, v=0), "crop_h -1": dict(i=7, v=-1),
    "in_w -1": dict(i=2, v=-1), "col0 -1": dict(i=11, v=-1), "in_ld < 3 in_w": dict(i=1, v=29),
    "row too short": dict(i=9, v=19), "plane too small": dict(i=10, v=119),
}


@pytest.mark.parametrize("what", sorted(_STORE_BAD))
def test_model_input_store_refuses_bad_arguments(what):
    from visualcloze_b200 import _lib
    args = list(_STORE_OK)
    args[_STORE_BAD[what]["i"]] = _STORE_BAD[what]["v"]
    assert _lib.lib().vcb_u8_to_model_input(*args, None) != 0
    assert _lib.lib().vcb_last_error().startswith(b"u8_to_model_input:")


def test_good_arguments_get_past_the_checks_without_a_device():
    """The same arguments with nothing wrong reach the device check (and only fail there when no GPU is present); an empty
    image with a NULL pointer is a blank cell, not an error."""
    from visualcloze_b200 import _lib
    if torch.cuda.is_available():
        pytest.skip("with a device the call would launch on the fake pointers")
    lib = _lib.lib()
    assert lib.vcb_resample_u8(*_RESAMPLE_OK, None) != 0 and b"CUDA" in lib.vcb_last_error()
    assert lib.vcb_u8_to_model_input(*_STORE_OK, None) != 0 and b"CUDA" in lib.vcb_last_error()
    blank = list(_STORE_OK)
    blank[0], blank[2], blank[3] = None, 0, 0
    assert lib.vcb_u8_to_model_input(*blank, None) != 0 and b"CUDA" in lib.vcb_last_error()
