"""The element-by-element checkers of tests/kernel_contract_ref.py, tested on the CPU: each accepts the emulated kernel output and
agrees with the oracle's rounding points, and each rejects the small errors that the rel-L2 bounds of test_kernels_gpu.py let
through (an injected error is applied to an emulated output; the rel-L2 of the mutation is asserted below that bound too, so the
test shows the gap it closes)."""
import math

import pytest
import torch

import kernel_contract_ref as kr
from conftest import rel_l2

BF16, F32 = torch.bfloat16, torch.float32
GRAIN = 2.0 ** -5                       # a in {-7..7} 2^-2, w in {-7..7} 2^-3


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _gemm_operands(M, N, K, seed=0):
    g = _gen(seed)
    a, w = kr.exact_bf16((M, K), g, 2), kr.exact_bf16((N, K), g, 3)
    bias = torch.randn(N, generator=g)
    return a, w, bias, kr.exact_acc(a, w, GRAIN)


def _canvas(vals: torch.Tensor, top=3, left=8, right=16, bottom=2, dtype=BF16):
    """the expected buffer: canaries everywhere, vals at [top:, left:]"""
    R, N = vals.shape
    buf = kr.canary_like(top + R + bottom, left + N + right, dtype)
    buf[top:top + R, left:left + N] = vals
    return buf


# ----------------------------------------------------------------------------------------------
# GEMM checkers
# ----------------------------------------------------------------------------------------------
def test_exact_operands_make_the_accumulator_order_independent():
    a, w, _, acc = _gemm_operands(64, 48, 1000)
    perm = torch.randperm(1000, generator=_gen(1))
    acc2 = (a.float()[:, perm] @ w.float()[:, perm].T)                     # another summation order, fp32
    assert torch.equal(acc, acc2)
    split = a.float()[:, :512] @ w.float()[:, :512].T + a.float()[:, 512:] @ w.float()[:, 512:].T   # split-K fold
    assert torch.equal(acc, split)
    with pytest.raises(AssertionError):
        kr.exact_acc(torch.full((1, 400000), 7 * 0.25, dtype=BF16), torch.full((1, 400000), 7 * 0.125, dtype=BF16), GRAIN)


def test_bias_checker_rejects_what_rel_l2_lets_through():
    """test_gemm_bias at 3456 x 3072 (rel-L2 bound 3e-3): one thread's 8 columns without the bias, and the 64 rows of one
    consumer warpgroup of one tile off by a factor of 1 + 2^-8 (K shortened: the checker does not depend on it)"""
    M, N, K = 3456, 3072, 64
    a, w, bias, acc = _gemm_operands(M, N, K)
    want = _canvas(kr.epi_bias(acc, bias))
    assert kr.check_exact(want.clone(), want) is None
    bad = kr.epi_bias(acc, bias)
    bad[M - 1, N - 8:] = acc[M - 1, N - 8:].to(BF16)
    assert rel_l2(bad, kr.epi_bias(acc, bias)) < 3e-3
    assert kr.check_exact(_canvas(bad), want) is not None
    bad = kr.epi_bias(acc, bias)
    bad[M - 64:] = (bad[M - 64:].float() * (1 + 2 ** -8)).to(BF16)
    assert rel_l2(bad, kr.epi_bias(acc, bias)) < 3e-3
    assert kr.check_exact(_canvas(bad), want) is not None


def test_gate_res_checker_pins_both_inner_roundings():
    """test_gemm_gate_residual_batched's shape (bound 4e-3): skipping both inner bf16 roundings changes ~27 % of the elements"""
    B, Lb, H, K = 2, 150, 512, 256
    a, w, bias, acc = _gemm_operands(B * Lb, H, K, seed=2)
    g = _gen(3)
    gate, res = torch.randn(B, H, generator=g).to(BF16), torch.randn(B * Lb, H, generator=g).to(BF16)
    rows = gate.repeat_interleave(Lb, 0)
    want = kr.epi_gate_res(acc, bias, rows, res)
    # the oracle's chain (layers.py:190: x + gate * Linear(a) under autocast, every op in bf16) is the same thing
    lin = (acc + bias).to(BF16)
    assert torch.equal(want, res + rows * lin)
    no_rnd = (res.float() + rows.float() * (acc + bias)).to(BF16)
    assert rel_l2(no_rnd, want) < 4e-3 and (no_rnd != want).float().mean() > 0.05
    assert kr.check_exact(_canvas(no_rnd), _canvas(want)) is not None
    wrong_gate = kr.epi_gate_res(acc, bias, gate[[0, 0]].repeat_interleave(Lb, 0), res)       # sample 1 reads sample 0's gate row
    assert kr.check_exact(_canvas(wrong_gate), _canvas(want)) is not None
    assert torch.equal(kr.epi_gate_res(acc, bias, None, res), (res.float() + lin.float()).to(BF16))


def test_checker_rejects_a_dropped_k_tail():
    M, N, K = 130, 72, 1000
    a, w, bias, acc = _gemm_operands(M, N, K, seed=4)
    short = kr.exact_acc(a[:, :960], w[:, :960], GRAIN)                     # the last partial k-block (40 of 64) dropped
    assert kr.check_exact(_canvas(kr.epi_bias(short, bias)), _canvas(kr.epi_bias(acc, bias))) is not None


def test_checker_rejects_rows_shifted_under_out_row_offset_and_a_lost_canary():
    M, N, K = 70, 13, 72
    a, w, bias, acc = _gemm_operands(M, N, K, seed=5)
    vals = kr.epi_bias(acc, bias)
    # N % 8 != 0: the kernel writes the round-up columns [N, 16) with the epilogue of a zero accumulator without bias: +0
    full = torch.cat([vals, torch.zeros(M, 3, dtype=BF16)], 1)
    want = _canvas(full, top=5)
    assert kr.check_exact(want.clone(), want) is None
    assert kr.check_exact(_canvas(full, top=6), want) is not None                 # every row one further down
    got = want.clone()
    got[5 + 7, 8 + 16] = 0                                                        # one canary just past round_up(N, 8)
    assert kr.check_exact(got, want) is not None
    got = want.clone()
    got[5 + 7, 8 + 14] = kr.canary_like(1, 1, BF16)[0, 0]                          # one round-up column not written
    assert kr.check_exact(got, want) is not None
    region = torch.zeros(want.shape, dtype=torch.bool)
    region[5:5 + M, 8:8 + N] = True
    assert kr.check_no_canary(want, region) is None and kr.check_no_canary(kr.canary_like(*want.shape, BF16), region) is not None


def test_bias_f32_checker():
    M, N, K = 40, 261, 72
    a, w, bias, acc = _gemm_operands(M, N, K, seed=6)
    vals = torch.cat([kr.epi_bias_f32(acc, bias), torch.zeros(M, 3)], 1)          # round_up(261, 4) = 264
    want = _canvas(vals, dtype=F32)
    assert kr.check_exact(want.clone(), want) is None
    got = want.clone()
    got[3 + 1, 8 + 5] = torch.nextafter(got[3 + 1, 8 + 5], torch.tensor(math.inf))
    assert kr.check_exact(got, want) is not None


def test_bias_f32_round_up_stops_at_a_multiple_of_4():
    """fp32 output, N % 8 in 1..4: the kernel's second float4 store is skipped, so the +0 columns end at round_up(N, 4) and the
    columns [round_up(N, 4), round_up(N, 8)) keep their canaries; a store of both float4s is rejected"""
    M, N, K = 40, 258, 72
    a, w, bias, acc = _gemm_operands(M, N, K, seed=16)
    vals = torch.cat([kr.epi_bias_f32(acc, bias), torch.zeros(M, 2)], 1)          # round_up(258, 4) = 260
    want = _canvas(vals, dtype=F32)
    assert kr.check_exact(want.clone(), want) is None
    assert bool(kr.bits(want[3:3 + M, 8 + 260:8 + 264]).eq(kr.CANARY_F32).all())
    both = want.clone()
    both[3:3 + M, 8 + 260:8 + 264] = 0.0                                           # the second float4 stored as well
    assert kr.check_exact(both, want) is not None


def test_gelu_interval_accepts_the_oracle_and_the_emulation_and_rejects_a_skipped_rounding():
    M, N, K = 200, 256, 72
    a, w, bias, acc = _gemm_operands(M, N, K, seed=7)
    bias = bias * 4
    lin = kr.linear_bf16(acc, bias)
    lo, hi = kr.epi_gelu_interval(acc, bias)
    region = torch.ones(M, N, dtype=torch.bool)
    # the reference's op on the bf16 Linear output, where its fp32 evaluation is accurate: below x = -3 torch's 1 + tanh(u)
    # cancels (relative error > 2^-16), the kernel's x / (1 + exp(-2u)) does not
    oracle = torch.nn.functional.gelu(lin.to(BF16), approximate="tanh")
    assert kr.check_interval(torch.where(lin > -3, oracle, lo), lo, hi, region & (lin > -3)) is None
    assert kr.check_interval(kr.gelu_emulated(lin), lo, hi, region) is None
    assert (hi != lo).float().mean() < 0.1                     # the interval is one bf16 value for most elements
    skipped = torch.nn.functional.gelu(acc + bias, approximate="tanh").to(BF16)    # bf16(acc + bias) skipped
    assert kr.check_interval(skipped, lo, hi, region) is not None
    flo, fhi = kr.gelu_interval(acc + bias, fast=True)                              # e4m3 form: fp32 input, tanh.approx
    assert kr.check_interval(torch.nn.functional.gelu(acc + bias, approximate="tanh").to(BF16), flo, fhi, region) is None


def test_qkv_interval_accepts_the_oracle_chain():
    """the oracle's rms_norm + apply_rope (oracle/flux_oracle.py, the chain _qkv_reference in test_kernels_gpu.py builds) on the
    same Linear output lies inside the QKV interval; a skipped bf16(x * rrms) rounding or a swapped RoPE sign does not"""
    from oracle import flux_oracle as fo
    L, H, K = 96, 256, 72
    heads = H // 128
    a, w, bias, acc = _gemm_operands(L, 3 * H, K, seed=8)
    g = _gen(9)
    qs, ks = (1 + 0.1 * torch.randn(128, generator=g)).to(BF16), (1 + 0.1 * torch.randn(128, generator=g)).to(BF16)
    ang = torch.randn(L, 64, generator=g) * 3
    cos, sin = torch.cos(ang), torch.sin(ang)
    lin = kr.linear_bf16(acc, bias)
    lo, hi = kr.qkv_interval(lin, qs, ks, cos, sin, H)
    region = torch.ones(L, 3 * H, dtype=torch.bool)

    def chain(norm):
        q, k, v = fo._split_heads(lin.to(BF16)[None], heads)
        q = fo.apply_rope(norm(q, qs), cos[None], sin[None])
        k = fo.apply_rope(norm(k, ks), cos[None], sin[None])
        return torch.cat([t.permute(0, 2, 1, 3).reshape(L, -1) for t in (q, k, v)], dim=-1)

    assert kr.check_interval(chain(fo.rms_norm), lo, hi, region) is None
    assert (hi.float() - lo.float()).abs().max() > 0 and (hi == lo).float().mean() > 0.5

    def no_round(x, scale):
        xf = x.float()
        return ((xf * torch.rsqrt((xf * xf).mean(-1, keepdim=True) + 1e-6)) * scale.float()).to(x.dtype)
    assert kr.check_interval(chain(no_round), lo, hi, region) is not None
    assert kr.check_interval(chain(fo.rms_norm), *kr.qkv_interval(lin, qs, ks, cos, -sin, H), region) is not None


# ----------------------------------------------------------------------------------------------
# attention bound
# ----------------------------------------------------------------------------------------------
def _qkv_attn(L, seed):
    g = _gen(seed)
    x = torch.randn(3, L, 128, generator=g)
    for i, s in ((0, 1.3), (1, 0.9)):
        x[i] = s * x[i] / x[i].pow(2).mean(-1, keepdim=True).sqrt()
    return x.to(BF16)


@pytest.mark.parametrize("L,seqlen", [(300, 300), (1000, 1000), (300, 129), (2, 2)])
def test_attention_bound_accepts_the_emulation_and_the_oracle(L, seqlen):
    from oracle import flux_oracle as fo
    q, k, v = _qkv_attn(L, seed=L + seqlen)
    o, bound = kr.attention_ref(q[:seqlen], k, v, seqlen)
    assert kr.check_attention(kr.attention_emulated(q[:seqlen], k, v, seqlen), o, bound) is None
    mask = torch.zeros(1, L, dtype=torch.int32)
    mask[0, :seqlen] = 1
    ones, zeros = torch.ones(1, L, 64), torch.zeros(1, L, 64)
    ref = fo.joint_attention(q[None, None], k[None, None], v[None, None], ones, zeros, mask, fo.Numerics("cuda_bf16"))[0]
    assert kr.check_attention(ref[:seqlen], o, bound) is None
    A = torch.softmax((q[:seqlen].double() @ k[:seqlen].double().T) * kr.SCALE, -1) @ v[:seqlen].double().abs()
    assert float((bound / (A + o.abs())).median()) < 2.0 ** -6        # ~2^-8 of sum p|v| + half an ulp: not a loose tolerance


def test_attention_bound_rejects_a_dropped_key_tile_a_padded_key_and_the_wrong_scale():
    L, n = 300, 260
    q, k, v = _qkv_attn(L, seed=11)
    o, bound = kr.attention_ref(q[:n], k, v, n)
    good = kr.attention_emulated(q[:n], k, v, n)
    assert kr.check_attention(good, o, bound) is None
    # one query row loses its second key tile (keys 128..255)
    keep = torch.cat([torch.arange(128), torch.arange(256, n)])
    dropped = good.clone()
    dropped[17] = kr.attention_emulated(q[17:18], k[keep], v[keep], keep.numel())[0]
    assert kr.check_attention(dropped, o, bound) is not None
    # one padded key (row n) included
    assert kr.check_attention(kr.attention_emulated(q[:n], k, v, n + 1), o, bound) is not None
    # 1 / sqrt(64) in place of 1 / sqrt(128)
    assert kr.check_attention(kr.attention_emulated(q[:n], k, v, n, scale=64 ** -0.5), o, bound) is not None


def test_directed_bf16_rounding():
    x = torch.tensor([1.0 + 2 ** -9, -1.0 - 2 ** -9, 0.0, 1e-42, -3.0, 2 ** -133], dtype=torch.float64)
    lo, hi = kr.bf16_down(x), kr.bf16_up(x)
    assert bool((lo.double() <= x).all() and (hi.double() >= x).all())
    assert float(lo[0]) == 1.0 and float(hi[0]) == 1.0 + 2 ** -7 and float(hi[1]) == -1.0 and float(lo[1]) == -1.0 - 2 ** -7
    assert float(lo[4]) == float(hi[4]) == -3.0


def test_attention_bound_holds_for_the_bf16_rounding_of_p_at_its_worst():
    """P's bf16 rounding costs up to 2^-8 of p (half an ulp just above a power of two), not 2^-9: with two keys at p = (1, 0.3622)
    (0.3622 rounds to 0.3613) the kernel stored -0.5859375 where the fp64 result is -0.5894, 3.5e-3 away -- outside a bound
    built on 2^-9, inside the derived one.  Same inputs as test_attention_contract[2-...] (L = 2, head 1 of 3, seed 2)."""
    g = torch.Generator().manual_seed(2)
    x = torch.randn(2, 3, 3, 128, generator=g)
    for i, s in ((0, 1.3), (1, 0.9)):
        x[:, i] = s * x[:, i] / x[:, i].pow(2).mean(-1, keepdim=True).sqrt()
    x = x.to(BF16)
    q, k, v = x[:, 0, 1], x[:, 1, 1], x[:, 2, 1]
    o, bound = kr.attention_ref(q, k, v, 2)
    got = kr.attention_emulated(q, k, v, 2)
    assert float(got[0, 91]) == -0.5859375
    assert kr.check_attention(got, o, bound) is None
