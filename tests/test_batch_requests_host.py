"""CPU checks of batched requests: the bucketing rule, the default batch table, the token count of a grid, the diffusers adapter's
argument mapping (lists, num_images_per_prompt, generator lists) on a fake model, and the ctypes prototypes and argument refusals of
the per-sample first-block-cache entry points."""
import ctypes as C
import math
import re

import pytest
import torch
from PIL import Image

from conftest import REPO


# ---- bucketing --------------------------------------------------------------------------------------------------------------------
def test_equal_token_counts_share_a_solve_in_order():
    from visualcloze_b200.pipeline import bucket_requests
    assert bucket_requests([3456, 1152, 3456, 1152, 3456], 8) == [[0, 2, 4], [1, 3]]
    assert bucket_requests([7], 1) == [[0]]
    assert bucket_requests([], 4) == []


def test_max_batch_splits_a_bucket_and_keeps_order():
    from visualcloze_b200.pipeline import bucket_requests
    assert bucket_requests([5] * 5, 2) == [[0, 1], [2, 3], [4]]
    assert bucket_requests([1, 2, 1, 2, 1, 1], 3) == [[0, 2, 4], [5], [1, 3]]
    assert bucket_requests([1, 2, 1], 1) == [[0], [2], [1]]
    got = bucket_requests([4, 4, 9, 4, 9, 4, 4], 2)
    assert sorted(i for b in got for i in b) == list(range(7))
    assert all(b == sorted(b) for b in got)


@pytest.mark.parametrize("bad", [0, -1, 1.5, "2", True, None])
def test_max_batch_is_validated(bad):
    from visualcloze_b200.pipeline import bucket_requests
    with pytest.raises(ValueError):
        bucket_requests([1, 1], bad)


def test_default_max_batch_table():
    from visualcloze_b200.pipeline import DEFAULT_MAX_BATCH, default_max_batch
    tops = [t for t, _ in DEFAULT_MAX_BATCH]
    assert tops == sorted(tops) and all(b >= 1 for _, b in DEFAULT_MAX_BATCH)
    for top, b in DEFAULT_MAX_BATCH:
        assert default_max_batch(top) == b
    assert default_max_batch(10 ** 9) == 1


def test_grid_tokens_match_the_rows_the_pipeline_builds():
    """2x3 and 3x2 at 384 both give 3456 tokens (so they share a solve); 1x2 gives 1152."""
    from visualcloze_b200.pipeline import grid_plan, grid_tokens
    sq = (384, 384)
    for (gh, gw), want in (((2, 3), 3456), ((3, 2), 3456), ((1, 2), 1152), ((2, 2), 2304)):
        sizes = [[sq] * gw for _ in range(gh)]
        sizes[-1][-1] = None
        cells, _, _ = grid_plan(sizes, gh, gw, 384)
        assert grid_tokens(cells, gh, gw) == want, (gh, gw)


def test_sdedit_size_is_the_solo_rule():
    from visualcloze_b200.pipeline import _sdedit_size
    assert _sdedit_size(None) == (1024, 1024)
    assert _sdedit_size((80, 96)) == (80, 96)
    assert _sdedit_size((90, 100)) == (80, 96)
    w, h = _sdedit_size((2048, 1024))
    assert w * h <= 1024 * 1024 and w % 16 == 0 and h % 16 == 0


# ---- adapter ----------------------------------------------------------------------------------------------------------------------
class _FakeModel:
    max_length = 512

    def __init__(self):
        self.calls = []

    def set_grid_size(self, h, w):
        self.calls.append(("grid", h, w))

    def process_images(self, images, prompts, seed=0, cfg=30, **kw):
        self.calls.append(("solo", prompts, seed, cfg, kw))
        return [Image.new("RGB", (32, 32))]

    def process_images_batch(self, requests, max_batch=None, **kw):
        self.calls.append(("batch", requests, max_batch, kw))
        return [[Image.new("RGB", (32, 32))] for _ in requests]


def _grid(rows=2, cols=2):
    g = [[Image.new("RGB", (40, 40)) for _ in range(cols)] for _ in range(rows)]
    g[-1][-1] = None
    return g


def test_adapter_single_call_is_unchanged():
    from visualcloze_b200.diffusers_adapter import VisualClozePipelineAdapter
    m = _FakeModel()
    out = VisualClozePipelineAdapter(m)("task", "content", _grid(), generator=torch.Generator().manual_seed(42),
                                         num_inference_steps=7, some_diffusers_only_argument=1)
    assert m.calls[0] == ("grid", 2, 2)
    kind, prompts, seed, cfg, kw = m.calls[1]
    assert kind == "solo" and seed == 42 and cfg == 30.0 and kw["steps"] == 7 and not kw["is_upsampling"]
    assert prompts == ["A grid layout with 2 rows and 2 columns, displaying 4 images arranged side by side.", "task", "content"]
    assert len(out.images) == 1 and len(out.images[0]) == 1
    VisualClozePipelineAdapter(m)("task", None, _grid())
    assert m.calls[-1][1][2] == "" and m.calls[-1][2] == 0


def test_adapter_num_images_per_prompt_seeds_follow_the_generator():
    from visualcloze_b200.diffusers_adapter import VisualClozePipelineAdapter
    m = _FakeModel()
    out = VisualClozePipelineAdapter(m)("task", "content", _grid(), generator=torch.Generator().manual_seed(10),
                                         num_images_per_prompt=4, max_batch=2)
    kind, reqs, max_batch, _ = m.calls[-1]
    assert kind == "batch" and max_batch == 2 and len(reqs) == 4 and len(out.images) == 4
    assert [r["seed"] for r in reqs] == [10, 11, 12, 13]
    assert all(r["grid"] == (2, 2) and r["prompts"][1:] == ["task", "content"] for r in reqs)


def test_adapter_lists_of_prompts_and_grids():
    from visualcloze_b200.diffusers_adapter import VisualClozePipelineAdapter
    m = _FakeModel()
    gens = [torch.Generator().manual_seed(s) for s in (5, 9, 2, 7)]
    out = VisualClozePipelineAdapter(m)(["t0", "t1"], ["c0", None], [_grid(2, 2), _grid(1, 3)], generator=gens,
                                         num_images_per_prompt=2, guidance_scale=3.5)
    _, reqs, _, _ = m.calls[-1]
    assert [r["seed"] for r in reqs] == [5, 9, 2, 7]
    assert [r["grid"] for r in reqs] == [(2, 2), (2, 2), (1, 3), (1, 3)]
    assert [r["prompts"][1:] for r in reqs] == [["t0", "c0"]] * 2 + [["t1", ""]] * 2
    assert reqs[2]["prompts"][0].startswith("A grid layout with 1 rows and 3 columns")
    assert all(r["cfg"] == 3.5 for r in reqs) and len(out.images) == 4
    # one grid for several prompts is shared; one prompt for several grids likewise
    VisualClozePipelineAdapter(m)(["a", "b", "c"], "c", _grid())
    assert [r["prompts"][1] for r in m.calls[-1][1]] == ["a", "b", "c"] and [r["seed"] for r in m.calls[-1][1]] == [0, 0, 0]
    VisualClozePipelineAdapter(m)("a", "c", [_grid(), _grid(1, 2)])
    assert [r["grid"] for r in m.calls[-1][1]] == [(2, 2), (1, 2)]


def test_adapter_refusals():
    from visualcloze_b200.diffusers_adapter import VisualClozePipelineAdapter
    a = VisualClozePipelineAdapter(_FakeModel())
    with pytest.raises(ValueError):
        a(["a", "b"], ["c", "d", "e"], _grid())
    with pytest.raises(ValueError):
        a("a", "c", _grid(), generator=[torch.Generator()], num_images_per_prompt=2)
    for bad in (0, -1, 1.5, True):
        with pytest.raises(ValueError):
            a("a", "c", _grid(), num_images_per_prompt=bad)
    with pytest.raises(ValueError):
        a("a", "c", [[Image.new("RGB", (8, 8))], [None, None]])
    with pytest.raises(ValueError):
        a("a", "c", [])
    with pytest.raises(ValueError):
        a("a", "c", _grid(), max_sequence_length=256)


def test_process_images_batch_signature():
    import inspect
    from visualcloze_b200.pipeline import VisualClozeModel
    sig = inspect.signature(VisualClozeModel.process_images_batch).parameters
    assert list(sig)[:2] == ["self", "requests"]
    for name, default in (("steps", 30), ("upsampling_steps", 10), ("upsampling_noise", 0.4), ("is_upsampling", True), ("max_batch", None)):
        assert sig[name].kind is inspect.Parameter.KEYWORD_ONLY and sig[name].default == default


# ---- per-sample first-block cache: ctypes and refusals ----------------------------------------------------------------------------
def test_ctypes_prototypes_of_the_per_sample_entry_points():
    from visualcloze_b200 import _lib
    sig = _lib._OPTIONAL
    assert sig["vcb_flux_set_first_block_cache_ex"] == (C.c_int, [C.c_void_p, C.c_float, C.c_int32])
    assert sig["vcb_flux_cache_stats_per_sample"] == (C.c_int, [C.c_void_p, C.c_int32, C.POINTER(C.c_int32), C.POINTER(C.c_int32),
                                                                 C.POINTER(C.c_float)])
    header = open(f"{REPO}/include/vcb200.h").read()
    assert re.search(r"int vcb_flux_set_first_block_cache_ex\(vcb_flux\* f, float threshold, int32_t per_sample\);", header)
    assert re.search(r"int vcb_flux_cache_stats_per_sample\(const vcb_flux\* f, int32_t B, int32_t\* computed, int32_t\* skipped, "
                     r"float\* last_diff\);", header)
    assert int(re.search(r"#define VCB_ABI_VERSION (\d+)", header).group(1)) == 7
    lib = _lib.lib()
    for name in ("vcb_flux_set_first_block_cache_ex", "vcb_flux_cache_stats_per_sample"):
        assert getattr(lib, name).restype is C.c_int


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


def test_c_set_ex_refusals(engine):
    lib, h = engine
    for bad_t in (-1.0, float("nan"), float("inf")):
        assert lib.vcb_flux_set_first_block_cache_ex(h, bad_t, 1) != 0
        assert b"threshold" in lib.vcb_last_error()
    for bad_mode in (-1, 2, 7):
        assert lib.vcb_flux_set_first_block_cache_ex(h, 0.1, bad_mode) != 0
        assert b"per_sample" in lib.vcb_last_error()
    assert lib.vcb_flux_set_first_block_cache_ex(h, 0.1, 1) == 0
    fake = (C.c_void_p * 2)(16, 32)
    assert lib.vcb_flux_sp_attach(h, 2, 0, fake, fake, fake, C.c_void_p(64), 1000) != 0
    assert b"first-block cache" in lib.vcb_last_error()
    assert lib.vcb_flux_set_first_block_cache_ex(h, 0.0, 1) == 0
    assert lib.vcb_flux_sp_attach(h, 2, 0, fake, fake, fake, C.c_void_p(64), 1000) == 0
    assert lib.vcb_flux_set_first_block_cache_ex(h, 0.1, 1) != 0
    assert b"sequence-parallel" in lib.vcb_last_error()
    assert lib.vcb_flux_sp_attach(h, 1, 0, None, None, None, None, 0) == 0


def test_c_per_sample_stats_refusals(engine):
    lib, h = engine
    c, s, d = (C.c_int32 * 2)(), (C.c_int32 * 2)(), (C.c_float * 2)()
    assert lib.vcb_flux_cache_stats_per_sample(h, 2, c, s, d) != 0
    assert b"prepare" in lib.vcb_last_error()
    assert lib.vcb_flux_cache_stats_per_sample(h, 2, None, s, d) != 0
    assert lib.vcb_flux_cache_stats_per_sample(None, 2, c, s, d) != 0


def test_c_per_sample_workspace(engine):
    """per-sample mode adds only the per-sample decision words; per-batch mode is the workspace it always was"""
    lib, h = engine
    B, Li, Lt, E = 3, 300, 40, 4
    assert lib.vcb_flux_set_first_block_cache_ex(h, 0.1, 0) == 0
    per_batch = lib.vcb_flux_workspace_bytes(h, B, Li, Lt, E)
    assert lib.vcb_flux_set_first_block_cache(h, 0.1) == 0
    assert lib.vcb_flux_workspace_bytes(h, B, Li, Lt, E) == per_batch
    assert lib.vcb_flux_set_first_block_cache_ex(h, 0.1, 1) == 0
    assert 0 <= lib.vcb_flux_workspace_bytes(h, B, Li, Lt, E) - per_batch <= 1024


def test_python_per_sample_flag():
    from visualcloze_b200 import model as M
    p = M.FluxParams(in_channels=64, out_channels=64, vec_in_dim=32, context_in_dim=64, hidden_size=256, mlp_ratio=2.0, num_heads=2,
                     depth=1, depth_single_blocks=1, axes_dim=[16, 56, 56], theta=10_000, qkv_bias=True, guidance_embed=True)
    m = M.FluxLoraWrapper(lora_rank=16, params=p, device="cpu")
    assert m._fbc_per_sample is False
    m.enable_first_block_cache(0.1, per_sample=True)
    assert (m._fbc, m._fbc_per_sample) == (0.1, True)
    with pytest.raises(ValueError):
        m.enable_first_block_cache(0.1, per_sample=1)
    assert m._fbc_per_sample is True
    m.enable_first_block_cache(0.2)
    assert (m._fbc, m._fbc_per_sample) == (0.2, False)
    assert m.cache_stats(per_sample=True) == []
    assert m.cache_stats()["computed"] == 0 and math.isnan(m.cache_stats()["last_diff"])
