"""CPU checks of the opt-in first-block cache: threshold validation, the refusal of sequence parallelism in either order (Python
and C), the ctypes prototypes of the two new entry points, the workspace it adds, and ABI 7 left as it was."""
import ctypes as C
import inspect
import math
import re

import pytest

from conftest import REPO


def _small_model():
    from visualcloze_b200 import model as M
    p = M.FluxParams(in_channels=64, out_channels=64, vec_in_dim=32, context_in_dim=64, hidden_size=256, mlp_ratio=2.0, num_heads=2,
                     depth=1, depth_single_blocks=1, axes_dim=[16, 56, 56], theta=10_000, qkv_bias=True, guidance_embed=True)
    return M.FluxLoraWrapper(lora_rank=16, params=p, device="cpu")


class _FakeSP:
    world = 2


class _OneRank:
    world = 1


@pytest.mark.parametrize("bad", [-1e-3, -1, float("nan"), float("inf"), -float("inf"), "0.1", True, [0.1]])
def test_threshold_validation_rejects(bad):
    m = _small_model()
    m.enable_first_block_cache(0.05)
    with pytest.raises(ValueError):
        m.enable_first_block_cache(bad)
    assert m._fbc == 0.05, "a refused threshold leaves the previous setting"


def test_threshold_none_and_zero_mean_off():
    from visualcloze_b200.engine import first_block_cache_threshold
    m = _small_model()
    assert m._fbc == 0.0, "off by default"
    for on, expect in ((0.1, 0.1), (None, 0.0), (2, 2.0), (0, 0.0), (1e30, 1e30)):
        m.enable_first_block_cache(on)
        assert m._fbc == expect
    assert first_block_cache_threshold(None) == 0.0
    assert m.cache_stats() == {"computed": 0, "skipped": 0, "last_diff": pytest.approx(math.nan, nan_ok=True)}


def test_cache_refuses_sequence_parallel_in_either_order():
    m = _small_model()
    m.enable_sequence_parallel(_FakeSP())
    with pytest.raises(ValueError):
        m.enable_first_block_cache(0.1)
    assert m._fbc == 0.0
    m.enable_first_block_cache(None)                     # switching it off stays allowed
    m.enable_sequence_parallel(None)
    m.enable_first_block_cache(0.1)
    with pytest.raises(ValueError):
        m.enable_sequence_parallel(_FakeSP())
    assert m._sp is None
    m.enable_sequence_parallel(_OneRank())               # one rank is not sequence parallelism
    m.enable_sequence_parallel(None)


def test_visualcloze_model_takes_first_block_cache_keyword_only():
    from visualcloze_b200.pipeline import VisualClozeModel
    p = inspect.signature(VisualClozeModel.__init__).parameters["first_block_cache"]
    assert p.kind is inspect.Parameter.KEYWORD_ONLY and p.default is None


def test_ctypes_prototypes_of_the_new_symbols():
    from visualcloze_b200 import _lib
    sig = _lib._OPTIONAL
    assert sig["vcb_flux_set_first_block_cache"] == (C.c_int, [C.c_void_p, C.c_float])
    assert sig["vcb_flux_cache_stats"] == (C.c_int, [C.c_void_p, C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.POINTER(C.c_float)])
    header = open(f"{REPO}/include/vcb200.h").read()
    assert re.search(r"int vcb_flux_set_first_block_cache\(vcb_flux\* f, float threshold\);", header)
    assert re.search(r"int vcb_flux_cache_stats\(const vcb_flux\* f, int32_t\* computed, int32_t\* skipped, float\* last_diff\);", header)
    lib = _lib.lib()
    for name in ("vcb_flux_set_first_block_cache", "vcb_flux_cache_stats"):
        assert getattr(lib, name).restype is C.c_int


def test_abi_is_still_7():
    from visualcloze_b200 import _lib
    header = open(f"{REPO}/include/vcb200.h").read()
    assert int(re.search(r"#define VCB_ABI_VERSION (\d+)", header).group(1)) == 7
    assert _lib.ABI_VERSION == 7 and _lib.lib().vcb_abi_version() == 7


# ---- the C engine without a device: vcb_flux_create and the setters keep host state only ----------------------------------------
@pytest.fixture
def engine():
    from visualcloze_b200 import _lib
    lib = _lib.lib()
    cfg = _lib.FluxConfigC()
    cfg.in_channels, cfg.out_channels, cfg.vec_in_dim, cfg.context_in_dim = 64, 64, 32, 64
    cfg.hidden, cfg.mlp_hidden, cfg.heads, cfg.depth, cfg.depth_single = 256, 512, 2, 1, 1
    cfg.axes_dim[0], cfg.axes_dim[1], cfg.axes_dim[2] = 16, 56, 56
    cfg.guidance_embed, cfg.theta = 1, 10000.0
    dbl, sgl = (_lib.DoubleW * 1)(), (_lib.SingleW * 1)()
    w = _lib.FluxWeightsC()
    w.dbl, w.sgl = C.cast(dbl, C.POINTER(_lib.DoubleW)), C.cast(sgl, C.POINTER(_lib.SingleW))
    h = C.c_void_p()
    _lib.check(lib.vcb_flux_create(C.byref(cfg), C.byref(w), C.byref(h)), "vcb_flux_create")
    yield lib, h
    lib.vcb_flux_destroy(h)


def test_c_threshold_validation_and_stats(engine):
    lib, h = engine
    for bad in (-1.0, float("nan"), float("inf")):
        assert lib.vcb_flux_set_first_block_cache(h, bad) != 0
        assert b"threshold" in lib.vcb_last_error()
    assert lib.vcb_flux_set_first_block_cache(h, 0.0) == 0
    assert lib.vcb_flux_set_first_block_cache(h, 0.25) == 0
    c, s, d = C.c_int32(-1), C.c_int32(-1), C.c_float(0)
    assert lib.vcb_flux_cache_stats(h, C.byref(c), C.byref(s), C.byref(d)) == 0
    assert (c.value, s.value) == (0, 0) and math.isnan(d.value)
    assert lib.vcb_flux_cache_stats(h, None, C.byref(s), C.byref(d)) != 0


def test_c_refuses_sequence_parallel_in_either_order(engine):
    lib, h = engine
    fake = (C.c_void_p * 2)(16, 32)                     # never dereferenced by the attach itself
    assert lib.vcb_flux_set_first_block_cache(h, 0.1) == 0
    assert lib.vcb_flux_sp_attach(h, 2, 0, fake, fake, fake, C.c_void_p(64), 1000) != 0
    assert b"first-block cache" in lib.vcb_last_error()
    assert lib.vcb_flux_set_first_block_cache(h, 0.0) == 0
    assert lib.vcb_flux_sp_attach(h, 2, 0, fake, fake, fake, C.c_void_p(64), 1000) == 0
    assert lib.vcb_flux_set_first_block_cache(h, 0.1) != 0
    assert b"sequence-parallel" in lib.vcb_last_error()
    assert lib.vcb_flux_sp_attach(h, 1, 0, None, None, None, None, 0) == 0
    assert lib.vcb_flux_set_first_block_cache(h, 0.1) == 0


def test_c_workspace_counts_the_cache_only_when_on(engine):
    lib, h = engine
    B, Li, Lt, E, H = 2, 300, 40, 4, 256
    off = lib.vcb_flux_workspace_bytes(h, B, Li, Lt, E)
    assert lib.vcb_flux_set_first_block_cache(h, 0.1) == 0
    on = lib.vcb_flux_workspace_bytes(h, B, Li, Lt, E)
    # x0 / r_ref pair (bf16) + R (fp32) + the partial sums and the decision
    assert B * Li * H * 8 <= on - off <= B * Li * H * 8 + 64 * 1024, (off, on)
    assert lib.vcb_flux_set_first_block_cache(h, 0.0) == 0
    assert lib.vcb_flux_workspace_bytes(h, B, Li, Lt, E) == off
