"""CPU checks of the unmerged LoRA mode: mode selection and the combinations it refuses are decided when they are set, and the
library and its binding agree on ABI 7 (which grew vcb_gemm_args and vcb_linear_w)."""
import re

import pytest
import torch

from conftest import REPO


def _small_model():
    from visualcloze_b200 import model as M
    p = M.FluxParams(in_channels=64, out_channels=64, vec_in_dim=32, context_in_dim=64, hidden_size=256, mlp_ratio=2.0, num_heads=2,
                     depth=1, depth_single_blocks=1, axes_dim=[16, 56, 56], theta=10_000, qkv_bias=True, guidance_embed=True)
    return M.FluxLoraWrapper(lora_rank=16, params=p, device="cpu")


class _FakeSP:
    world = 2


def test_set_lora_mode_rejects_unknown_modes():
    m = _small_model()
    assert m.lora_mode == "merged"
    m.set_lora_mode("unmerged")
    assert m.lora_mode == "unmerged"
    m.set_lora_mode("merged")
    for bad in ("fused", "Unmerged", "", None):
        with pytest.raises(ValueError):
            m.set_lora_mode(bad)
    assert m.lora_mode == "merged"


@pytest.mark.parametrize("precision", ["fp8", "fp8_all"])
def test_unmerged_refuses_fp8_in_either_order(precision):
    m = _small_model()
    m.set_linear_precision(precision)
    with pytest.raises(ValueError):
        m.set_lora_mode("unmerged")
    assert m.lora_mode == "merged"
    m.set_linear_precision("bf16")
    m.set_lora_mode("unmerged")
    with pytest.raises(ValueError):
        m.set_linear_precision(precision)
    assert m.linear_precision == "bf16"


def test_unmerged_refuses_sequence_parallel_in_either_order():
    m = _small_model()
    m.enable_sequence_parallel(_FakeSP())
    with pytest.raises(ValueError):
        m.set_lora_mode("unmerged")
    m.enable_sequence_parallel(None)
    m.set_lora_mode("unmerged")
    with pytest.raises(ValueError):
        m.enable_sequence_parallel(_FakeSP())
    m.enable_sequence_parallel(None)              # switching it off stays allowed


def test_engine_rejects_bad_lora_mode_before_touching_the_device():
    from visualcloze_b200.engine import FluxEngine
    with pytest.raises(ValueError):
        FluxEngine(None, {}, lora_mode="fused")
    with pytest.raises(ValueError):
        FluxEngine(None, {}, fp8=1, lora_mode="unmerged")


def test_abi_version_is_7_on_both_sides():
    from visualcloze_b200 import _lib
    assert _lib.ABI_VERSION == 7
    header = open(f"{REPO}/include/vcb200.h").read()
    assert int(re.search(r"#define VCB_ABI_VERSION (\d+)", header).group(1)) == 7
    assert _lib.lib().vcb_abi_version() == 7
    names = [f[0] for f in _lib.GemmArgs._fields_]
    assert names[-6:] == ["lora_t", "ld_lora_t", "lora_t_batch_stride", "lora_b", "lora_rank", "alpha"]
    assert [f[0] for f in _lib.LinearW._fields_][-4:] == ["lora_a", "lora_b", "rank", "lora_scale"]


def test_visualcloze_model_takes_lora_mode_keyword_only():
    import inspect
    from visualcloze_b200.pipeline import VisualClozeModel
    p = inspect.signature(VisualClozeModel.__init__).parameters["lora_mode"]
    assert p.kind is inspect.Parameter.KEYWORD_ONLY and p.default == "merged"
