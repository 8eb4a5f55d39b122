"""The four AdaLN LayerNorm variants (bf16 / e4m3 output x statistics from a pass / from the producer) share one kernel body:
every variant's grouped launch equals two single launches, the e4m3 output is exactly the row-wise quantisation of the bf16
output taken from the same statistics source, and every entry point accepts the same hidden sizes."""
import pytest
import torch

pytestmark = pytest.mark.gpu

BF16 = torch.bfloat16
F8 = torch.float8_e4m3fn
MAX_HIDDEN = 6144


@pytest.fixture(scope="module")
def ops():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    from visualcloze_b200 import ops as _ops
    return _ops


def _slot_stats(x):
    """(sum, sum of squares) per row and per 64 columns, the layout the GATE_RES epilogue leaves behind"""
    xf = x.float().reshape(x.shape[0], x.shape[1] // 64, 64)
    return torch.stack((xf.sum(-1), (xf * xf).sum(-1)), dim=-1).contiguous()


# (bf16, pass) is test_kernels_gpu.py::test_ln_modulate_grouped_two_streams_one_launch
@pytest.mark.parametrize("out_dtype,stats_src", [("bf16", "producer"), ("e4m3", "pass"), ("e4m3", "producer")])
def test_grouped_launch_equals_two_single_launches(ops, out_dtype, stats_src):
    """img and txt streams of a double block (their own shift / scale, rows interleaved per sample in the joint buffer, blocks
    straddling samples) in ONE launch must equal two separate launches bit for bit, rows and per-row scales alike."""
    B, Lt, Li, H = 2, 24, 83, 512
    L = Lt + Li
    g = torch.Generator().manual_seed(61)
    x = (torch.randn(B * L, H, generator=g) * 2.0).to(BF16).cuda()
    mods = [(0.5 * torch.randn(B, 6 * H, generator=g)).to(BF16).cuda() for _ in range(2)]   # [B, 6H]: shift at col 0, scale at col H
    problems = [(Lt, B * Li, Li, mods[0][:, :H], mods[0][:, H:2 * H]), (0, B * Lt, Lt, mods[1][:, :H], mods[1][:, H:2 * H])]
    stats = _slot_stats(x) if stats_src == "producer" else None
    fp8 = out_dtype == "e4m3"
    ref, got = (torch.zeros(B * L, H, dtype=F8 if fp8 else BF16, device="cuda") for _ in range(2))
    ref_rs, got_rs = (torch.full((B * L,), -1.0, device="cuda") for _ in range(2))
    for p in problems:
        ops.ln_modulate_grouped(x, ref, [p], H, L, 6 * H, row_scale=ref_rs if fp8 else None, stats=stats)
    ops.ln_modulate_grouped(x, got, problems, H, L, 6 * H, row_scale=got_rs if fp8 else None, stats=stats)
    torch.cuda.synchronize()
    if fp8:
        ref, got = ref.view(torch.uint8), got.view(torch.uint8)
        assert torch.equal(got_rs, ref_rs)
        assert bool((ref_rs > 0).all())
    assert torch.equal(got, ref)
    assert float(ref.float().abs().max()) > 0


@pytest.mark.parametrize("grouped", [False, True])
@pytest.mark.parametrize("stats_src", ["pass", "producer"])
@pytest.mark.parametrize("H", [256, 3072, 4096, 5120])
def test_fp8_output_is_the_quantised_bf16_output(ops, H, stats_src, grouped):
    """row_scale == max(max|y_bf16|, 1e-12) * fp32(1 / 448) and y8 == e4m3(y_bf16 * (1 / row_scale)), bit for bit; the img and txt
    rows of a joint buffer (blocks straddle samples), img alone or both streams in one launch."""
    g = torch.Generator().manual_seed(H)
    B, Lt, Li = 2, 24, 83
    L = Lt + Li
    x = (torch.randn(B * L, H, generator=g) * 1.7 + 0.3).to(BF16).cuda()
    x[Lt + 5] = 0                                                  # a constant row: y = shift
    mods = [(0.4 * torch.randn(B, 6 * H, generator=g)).to(BF16).cuda() for _ in range(2)]
    problems = [(Lt, B * Li, Li, mods[0][:, :H], mods[0][:, H:2 * H]), (0, B * Lt, Lt, mods[1][:, :H], mods[1][:, H:2 * H])]
    if not grouped:
        problems = problems[:1]
    stats = _slot_stats(x) if stats_src == "producer" else None
    y = torch.zeros(B * L, H, dtype=BF16, device="cuda")
    y8 = torch.zeros(B * L, H, dtype=F8, device="cuda")
    rs = torch.full((B * L,), -1.0, device="cuda")
    ops.ln_modulate_grouped(x, y, problems, H, L, 6 * H, stats=stats)
    ops.ln_modulate_grouped(x, y8, problems, H, L, 6 * H, row_scale=rs, stats=stats)
    torch.cuda.synchronize()
    rows = torch.zeros(B * L, dtype=torch.bool, device="cuda")
    for off, n, rpb, _, _ in problems:
        for b in range(n // rpb):
            rows[b * L + off:b * L + off + rpb] = True
    assert bool((rs[~rows] == -1).all()), "rows outside the problems must not be touched"
    y, y8, rs = y[rows].float(), y8[rows], rs[rows]
    s_ref = y.abs().amax(dim=1).clamp_min(1e-12) * torch.tensor(1.0 / 448.0, device="cuda")
    assert torch.equal(rs, s_ref)
    ref8 = (y * (1 / rs)[:, None]).to(F8)
    assert torch.equal(y8.view(torch.uint8), ref8.view(torch.uint8))


def test_hidden_limit_is_shared(ops):
    """hidden = 6144 runs in all five entry points; 6400 (a multiple of 256 above the limit) is refused by each, by name."""
    rows = 40
    for H, ok in ((MAX_HIDDEN, True), (MAX_HIDDEN + 256, False)):
        g = torch.Generator().manual_seed(H)
        x = torch.randn(rows, H, generator=g).to(BF16).cuda()
        shift, scale = ((0.3 * torch.randn(1, H, generator=g)).to(BF16).cuda() for _ in range(2))
        stats = _slot_stats(x)
        y = torch.zeros(rows, H, dtype=BF16, device="cuda")
        y8 = torch.zeros(rows, H, dtype=F8, device="cuda")
        rs = torch.zeros(rows, device="cuda")
        half = [(0, rows // 2, rows // 2, shift, scale), (rows // 2, rows // 2, rows // 2, shift, scale)]
        calls = {
            "ln_modulate": lambda: ops.ln_modulate(x, shift, scale, y, rows_per_batch=rows),
            "ln_modulate_grouped": lambda: ops.ln_modulate_grouped(x, y, half, H, rows // 2, 0),
            "ln_modulate_stats": lambda: ops.ln_modulate_stats(x, shift, scale, y, stats, rows_per_batch=rows),
            "ln_modulate_fp8": lambda: ops.ln_modulate_fp8(x, shift, scale, y8, rs, rows_per_batch=rows),
            "ln_modulate_fp8_stats": lambda: ops.ln_modulate_fp8(x, shift, scale, y8, rs, rows_per_batch=rows, stats=stats),
        }
        for name, call in calls.items():
            if ok:
                y.zero_(); rs.zero_()
                call()
                torch.cuda.synchronize()
                assert float(y.float().abs().max()) > 0 or bool((rs > 0).all()), name
            else:
                with pytest.raises(Exception, match=f": {name}: hidden must be"):
                    call()
