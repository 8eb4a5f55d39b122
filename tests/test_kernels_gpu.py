"""Per-kernel parity on the H100: every test calls through the C ABI (visualcloze_b200.ops -> libvcb200.so)
and compares with the CPU oracle (oracle/flux_oracle.py) or, for the bare GEMM, a plain fp32 torch matmul of
the same bf16 operands.  Tolerances are stated per test."""
import math

import pytest
import torch

from conftest import rel_l2

pytestmark = pytest.mark.gpu

BF16 = torch.bfloat16


@pytest.fixture(scope="module")
def ops():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    from visualcloze_b200 import ops as _ops
    return _ops


def _randn(*shape, seed=0, scale=1.0, dtype=BF16):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(dtype)


def _stats(got, ref):
    got, ref = got.float().cpu(), ref.float().cpu()
    d = (got - ref).abs()
    return f"rel_l2={rel_l2(got, ref):.3e} max_abs={d.max().item():.3e} ref_absmax={ref.abs().max().item():.3e} " \
           f"nan={int(torch.isnan(got).sum())} argmax={tuple(int(i) for i in torch.unravel_index(d.argmax(), d.shape))}"


# ------------------------------------------------------------------------------------------------
# operand-layout probes (single wgmma tile)
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("ksteps", [4, 8])
def test_probe_kmajor_ss(ops, ksteps):
    K = 16 * ksteps
    a, b = _randn(128, K, seed=1), _randn(128, K, seed=2)
    out = ops.umma_probe(a.cuda(), b.cuda(), ksteps, False, False)
    ref = a.float() @ b.float().T
    assert rel_l2(out.cpu(), ref) < 1e-5, _stats(out, ref)


@pytest.mark.parametrize("ksteps", [4, 8])
def test_probe_b_mn_major(ops, ksteps):
    """B given as [K, N] with N contiguous (the V tile of attention)."""
    K = 16 * ksteps
    a, b = _randn(128, K, seed=3), _randn(K, 128, seed=4)
    out = ops.umma_probe(a.cuda(), b.cuda(), ksteps, True, False, b_lbo=K * 128, b_sbo=1024, b_kstep_bytes=2048)
    ref = a.float() @ b.float()
    assert rel_l2(out.cpu(), ref) < 1e-5, _stats(out, ref)


@pytest.mark.parametrize("ksteps", [4, 8])
def test_probe_a_from_tmem(ops, ksteps):
    """A fed from registers as packed bf16 pairs (the P tile of attention; the test keeps its first name), B MN-major."""
    K = 16 * ksteps
    a, b = _randn(128, K, seed=5), _randn(K, 128, seed=6)
    out = ops.umma_probe(a.cuda(), b.cuda(), ksteps, True, True, b_lbo=K * 128, b_sbo=1024, b_kstep_bytes=2048)
    ref = a.float() @ b.float()
    assert rel_l2(out.cpu(), ref) < 1e-5, _stats(out, ref)


def test_probe_a_from_tmem_b_kmajor(ops):
    a, b = _randn(128, 128, seed=7), _randn(128, 128, seed=8)
    out = ops.umma_probe(a.cuda(), b.cuda(), 8, False, True)
    ref = a.float() @ b.float().T
    assert rel_l2(out.cpu(), ref) < 1e-5, _stats(out, ref)


# ------------------------------------------------------------------------------------------------
# GEMM
# ------------------------------------------------------------------------------------------------
GEMM_SHAPES = [
    (128, 256, 64), (128, 256, 512), (200, 264, 384), (384, 768, 3072), (1000, 64, 3072), (29, 1536, 256),
    (3456, 3072, 3072),
]


@pytest.mark.parametrize("cta_group", [1, 2])
@pytest.mark.parametrize("block_n", [0, 128, 192, 256])
@pytest.mark.parametrize("shape", GEMM_SHAPES)
def test_gemm_bias(ops, shape, block_n, cta_group):
    M, N, K = shape
    a, w = _randn(M, K, seed=1), _randn(N, K, seed=2, scale=1 / math.sqrt(K))
    bias = _randn(N, seed=3, dtype=torch.float32)
    out = torch.full((M, N), 7.0, dtype=BF16, device="cuda")
    ops.gemm(a.cuda(), w.cuda(), bias.cuda(), out, block_n=block_n, cta_group=cta_group)
    torch.cuda.synchronize()
    ref = (a.float() @ w.float().T + bias).to(BF16)
    # fp32 accumulation both sides; difference = summation order + one bf16 rounding
    assert rel_l2(out.cpu(), ref) < 3e-3, _stats(out, ref)


def test_gemm_block64_and_strided_output(ops):
    M, N, K = 300, 64, 512
    a, w = _randn(M, K, seed=1), _randn(N, K, seed=2, scale=1 / math.sqrt(K))
    buf = torch.zeros(M, 256, dtype=BF16, device="cuda")
    ops.gemm(a.cuda(), w.cuda(), None, buf, out_col_offset=128, block_n=64, cta_group=1)
    ref = (a.float() @ w.float().T).to(BF16)
    assert rel_l2(buf[:, 128:192].cpu(), ref) < 3e-3, _stats(buf[:, 128:192], ref)
    assert float(buf[:, :128].abs().max()) == 0 and float(buf[:, 192:].abs().max()) == 0


@pytest.mark.parametrize("cta_group", [1, 2])
def test_gemm_gelu(ops, cta_group):
    M, N, K = 520, 1024, 256
    a, w = _randn(M, K, seed=1), _randn(N, K, seed=2, scale=1 / math.sqrt(K))
    bias = _randn(N, seed=3, dtype=torch.float32, scale=0.1)
    out = torch.empty(M, N, dtype=BF16, device="cuda")
    ops.gemm(a.cuda(), w.cuda(), bias.cuda(), out, epilogue=ops.EPI_BIAS_GELU, cta_group=cta_group)
    lin = (a.float() @ w.float().T + bias).to(BF16)
    ref = torch.nn.functional.gelu(lin, approximate="tanh")
    assert rel_l2(out.cpu(), ref) < 4e-3, _stats(out, ref)


@pytest.mark.parametrize("cta_group", [1, 2])
def test_gemm_gate_residual_batched(ops, cta_group):
    """x <- x + gate[b] * (attn @ W^T + bias), in place, two samples with their own gate rows (layers.py:190)."""
    B, Lb, H, K = 2, 150, 512, 256
    a, w = _randn(B * Lb, K, seed=1), _randn(H, K, seed=2, scale=1 / math.sqrt(K))
    bias = _randn(H, seed=3, dtype=torch.float32, scale=0.1)
    gate, x = _randn(B, H, seed=4), _randn(B * Lb, H, seed=5)
    xg = x.cuda().clone()
    ops.gemm(a.cuda(), w.cuda(), bias.cuda(), xg, epilogue=ops.EPI_GATE_RES, rows_per_batch=Lb, gate=gate.cuda(),
             res=xg, cta_group=cta_group)
    lin = (a.float() @ w.float().T + bias).to(BF16).reshape(B, Lb, H)
    ref = (x.reshape(B, Lb, H) + gate[:, None, :] * lin).reshape(B * Lb, H)
    assert rel_l2(xg.cpu(), ref) < 4e-3, _stats(xg, ref)


@pytest.mark.parametrize("cta_group", [0, 1, 2])
def test_gemm_grouped_two_streams(ops, cta_group):
    """img + txt streams of a double block in ONE launch: different A rows of a joint buffer, different weights, gates and
    row offsets; in-place gated residual (layers.py:190-195)."""
    B, Li, Lt, H, K = 2, 300, 40, 512, 256
    L = Li + Lt
    attn = _randn(B * L, K, seed=1)                                  # joint [B, L, K] buffer, txt rows first
    x = _randn(B * L, H, seed=2)
    w = [_randn(H, K, seed=3, scale=1 / math.sqrt(K)), _randn(H, K, seed=4, scale=1 / math.sqrt(K))]
    bias = [_randn(H, seed=5, dtype=torch.float32, scale=0.1), _randn(H, seed=6, dtype=torch.float32, scale=0.1)]
    gate = [_randn(B, H, seed=7), _randn(B, H, seed=8)]
    xg, ag = x.cuda().clone(), attn.cuda()
    probs = []
    for s, (rows, off) in enumerate(((Li, Lt), (Lt, 0))):           # img then txt
        probs.append(dict(a=ag[off:], w=w[s].cuda(), bias=bias[s].cuda(), out=xg, epilogue=ops.EPI_GATE_RES, m=B * rows,
                          rows_per_batch=rows, out_batch_rows=L, out_row_offset=off, a_batch_stride=L * K, gate=gate[s].cuda(),
                          res=xg, cta_group=cta_group))
    ops.gemm_grouped(probs[0], probs[1])
    torch.cuda.synchronize()
    ref = x.reshape(B, L, H).clone()
    a3 = attn.reshape(B, L, K)
    for s, (rows, off) in enumerate(((Li, Lt), (Lt, 0))):
        lin = (a3[:, off:off + rows].float() @ w[s].float().T + bias[s]).to(BF16)
        ref[:, off:off + rows] = x.reshape(B, L, H)[:, off:off + rows] + gate[s][:, None, :] * lin
    assert rel_l2(xg.cpu(), ref.reshape(B * L, H)) < 4e-3, _stats(xg, ref.reshape(B * L, H))


def _qkv_reference(a, w, bias, qs, ks, cos, sin, heads):
    from oracle import flux_oracle as fo
    L = a.shape[0]
    lin = (a.float() @ w.float().T + bias).to(BF16)[None]              # [1, L, 3H]
    q, k, v = fo._split_heads(lin, heads)
    q = fo.apply_rope(fo.rms_norm(q, qs), cos[None], sin[None])
    k = fo.apply_rope(fo.rms_norm(k, ks), cos[None], sin[None])
    return torch.cat([t.permute(0, 2, 1, 3).reshape(L, -1) for t in (q, k, v)], dim=-1)


@pytest.mark.parametrize("cta_group", [1, 2])
@pytest.mark.parametrize("block_n", [128, 256])
def test_gemm_qkv_epilogue(ops, block_n, cta_group):
    """bias + QK-RMSNorm + RoPE fused into the projection (layers.py:165-174, math.py:112-117), written at a row
    offset of a joint txt||img buffer."""
    L, H, heads, K, row_off, Ltot = 200, 256, 2, 256, 24, 256
    a, w = _randn(L, K, seed=1), _randn(3 * H, K, seed=2, scale=1 / math.sqrt(K))
    bias = _randn(3 * H, seed=3, dtype=torch.float32, scale=0.1)
    qs, ks = (1 + 0.1 * _randn(128, seed=4, dtype=torch.float32)).to(BF16), (1 + 0.1 * _randn(128, seed=5, dtype=torch.float32)).to(BF16)
    ang = _randn(Ltot, 64, seed=6, dtype=torch.float32) * 3
    cos, sin = torch.cos(ang), torch.sin(ang)
    rope = torch.stack([cos, sin], -1).permute(1, 0, 2).contiguous()      # pair-major [64, rows, 2]
    out = torch.zeros(Ltot, 3 * H, dtype=BF16, device="cuda")
    ops.gemm(a.cuda(), w.cuda(), bias.cuda(), out, epilogue=ops.EPI_QKV, hidden=H, q_scale=qs.cuda(), k_scale=ks.cuda(),
             rope=rope.cuda(), rows_per_batch=L, out_batch_rows=Ltot, out_row_offset=row_off, block_n=block_n,
             cta_group=cta_group)
    ref = _qkv_reference(a, w, bias, qs, ks, cos[row_off:row_off + L], sin[row_off:row_off + L], heads)
    got = out[row_off:row_off + L].cpu()
    assert rel_l2(got, ref) < 6e-3, _stats(got, ref)
    assert float(out[:row_off].abs().max()) == 0 and float(out[row_off + L:].abs().max()) == 0


@pytest.mark.parametrize("cta_group", [1, 2])
def test_gemm_streamk_fewer_tiles_than_ctas(ops, cta_group):
    """One partial wave (M = 600, N = 3072: 36 pair tiles / 60 single tiles on 74 / 148 slots) with a long K: with stream-K
    (VCB_STREAMK=1, or the auto policy) every CTA gets an equal K range of the few tiles; results must match either way."""
    M, N, K = 600, 3072, 8192
    a, w = _randn(M, K, seed=1), _randn(N, K, seed=2, scale=1 / math.sqrt(K))
    bias = _randn(N, seed=3, dtype=torch.float32, scale=0.1)
    gate, x = _randn(1, N, seed=4), _randn(M, N, seed=5)
    out = x.cuda().clone()
    ops.gemm(a.cuda(), w.cuda(), bias.cuda(), out, epilogue=ops.EPI_GATE_RES, gate=gate.cuda(), res=out, cta_group=cta_group, block_n=256)
    torch.cuda.synchronize()
    ref = x + gate * (a.float() @ w.float().T + bias).to(BF16)
    assert rel_l2(out.cpu(), ref) < 4e-3, _stats(out, ref)


@pytest.mark.parametrize("cta_group", [1, 2])
@pytest.mark.parametrize("epi", ["qkv", "gelu", "gate"])
def test_gemm_streamk_multiwave(ops, epi, cta_group):
    """More tiles than CTA pairs and a non-integral wave count.  With VCB_STREAMK=1 in the environment the partial last wave
    is split along K (fp32 partials through the workspace); results must match the reference either way, for every epilogue."""
    M, K, H, heads = 3000, 512, 1024, 8
    a = _randn(M, K, seed=1)
    if epi == "qkv":
        w = _randn(3 * H, K, seed=2, scale=1 / math.sqrt(K))
        bias = _randn(3 * H, seed=3, dtype=torch.float32, scale=0.1)
        qs, ks = (1 + 0.1 * _randn(128, seed=4, dtype=torch.float32)).to(BF16), (1 + 0.1 * _randn(128, seed=5, dtype=torch.float32)).to(BF16)
        ang = _randn(M, 64, seed=6, dtype=torch.float32) * 3
        cos, sin = torch.cos(ang), torch.sin(ang)
        rope = torch.stack([cos, sin], -1).permute(1, 0, 2).contiguous()
        out = torch.zeros(M, 3 * H, dtype=BF16, device="cuda")
        ops.gemm(a.cuda(), w.cuda(), bias.cuda(), out, epilogue=ops.EPI_QKV, hidden=H, q_scale=qs.cuda(), k_scale=ks.cuda(),
                 rope=rope.cuda(), cta_group=cta_group)
        ref = _qkv_reference(a, w, bias, qs, ks, cos, sin, heads)
        tol = 6e-3
    else:
        N = 3072
        w = _randn(N, K, seed=2, scale=1 / math.sqrt(K))
        bias = _randn(N, seed=3, dtype=torch.float32, scale=0.1)
        lin = (a.float() @ w.float().T + bias).to(BF16)
        if epi == "gelu":
            out = torch.empty(M, N, dtype=BF16, device="cuda")
            ops.gemm(a.cuda(), w.cuda(), bias.cuda(), out, epilogue=ops.EPI_BIAS_GELU, cta_group=cta_group)
            ref = torch.nn.functional.gelu(lin, approximate="tanh")
        else:
            gate, x = _randn(1, N, seed=4), _randn(M, N, seed=5)
            out = x.cuda().clone()
            ops.gemm(a.cuda(), w.cuda(), bias.cuda(), out, epilogue=ops.EPI_GATE_RES, gate=gate.cuda(), res=out, cta_group=cta_group)
            ref = x + gate * lin
        tol = 4e-3
    torch.cuda.synchronize()
    assert rel_l2(out.cpu(), ref) < tol, _stats(out, ref)


@pytest.mark.parametrize("cta_group", [1, 2])
def test_gemm_linear1_epilogue(ops, cta_group):
    """single-stream linear1: qkv columns get norm+rope, mlp columns get GELU into the linear2 input (layers.py:235-244)."""
    L, H, heads, mlp = 160, 256, 2, 512
    a, w = _randn(L, H, seed=1), _randn(3 * H + mlp, H, seed=2, scale=1 / math.sqrt(H))
    bias = _randn(3 * H + mlp, seed=3, dtype=torch.float32, scale=0.1)
    qs, ks = (1 + 0.1 * _randn(128, seed=4, dtype=torch.float32)).to(BF16), (1 + 0.1 * _randn(128, seed=5, dtype=torch.float32)).to(BF16)
    ang = _randn(L, 64, seed=6, dtype=torch.float32) * 3
    cos, sin = torch.cos(ang), torch.sin(ang)
    rope = torch.stack([cos, sin], -1).permute(1, 0, 2).contiguous()
    qkv = torch.zeros(L, 3 * H, dtype=BF16, device="cuda")
    cat = torch.zeros(L, H + mlp, dtype=BF16, device="cuda")
    ops.gemm(a.cuda(), w.cuda(), bias.cuda(), qkv, epilogue=ops.EPI_LINEAR1, hidden=H, q_scale=qs.cuda(), k_scale=ks.cuda(),
             rope=rope.cuda(), out2=cat, out2_col_offset=H, cta_group=cta_group)
    ref_qkv = _qkv_reference(a, w[:3 * H], bias[:3 * H], qs, ks, cos, sin, heads)
    lin = (a.float() @ w[3 * H:].float().T + bias[3 * H:]).to(BF16)
    ref_mlp = torch.nn.functional.gelu(lin, approximate="tanh")
    assert rel_l2(qkv.cpu(), ref_qkv) < 6e-3, _stats(qkv, ref_qkv)
    assert rel_l2(cat[:, H:].cpu(), ref_mlp) < 4e-3, _stats(cat[:, H:], ref_mlp)
    assert float(cat[:, :H].abs().max()) == 0


@pytest.mark.parametrize("cta_group", [1, 2])
@pytest.mark.parametrize("epi", ["qkv", "linear1"])
def test_gemm_sequence_parallel_head_routing(ops, epi, cta_group):
    """Sequence-parallel epilogue (SURVEY.md 8f-2): the q/k/v columns of head h land in rank h // (heads/W)'s buffer
    [W * rows, 3H/W] at row sp_row_offset + output row, through staged TMA tile stores (here both "ranks" are local buffers).
    L = 300 leaves a partial second M tile: the TMA unit must clip the rows past the problem's extent."""
    W, rank, L, H, heads, K, row_off, Ltot, mlp = 2, 1, 300, 512, 4, 256, 24, 340, 384
    hw = H // W
    N = 3 * H + (mlp if epi == "linear1" else 0)
    a, w = _randn(L, K, seed=1), _randn(N, K, seed=2, scale=1 / math.sqrt(K))
    bias = _randn(N, seed=3, dtype=torch.float32, scale=0.1)
    qs, ks = (1 + 0.1 * _randn(128, seed=4, dtype=torch.float32)).to(BF16), (1 + 0.1 * _randn(128, seed=5, dtype=torch.float32)).to(BF16)
    ang = _randn(Ltot, 64, seed=6, dtype=torch.float32) * 3
    cos, sin = torch.cos(ang), torch.sin(ang)
    rope = torch.stack([cos, sin], -1).permute(1, 0, 2).contiguous()
    bufs = [torch.zeros(W * Ltot, 3 * hw, dtype=BF16, device="cuda") for _ in range(W)]
    local = torch.zeros(Ltot, 3 * H, dtype=BF16, device="cuda")          # `out` is not written for q/k/v columns in this mode
    cat = torch.zeros(Ltot, H + mlp, dtype=BF16, device="cuda")
    kw = dict(out2=cat, out2_col_offset=H) if epi == "linear1" else {}
    ops.gemm(a.cuda(), w.cuda(), bias.cuda(), local, epilogue=ops.EPI_LINEAR1 if epi == "linear1" else ops.EPI_QKV, hidden=H,
             q_scale=qs.cuda(), k_scale=ks.cuda(), rope=rope.cuda(), rows_per_batch=L, out_batch_rows=Ltot, out_row_offset=row_off,
             cta_group=cta_group, sp_out=bufs, sp_row_offset=rank * Ltot, **kw)
    torch.cuda.synchronize()
    ref = _qkv_reference(a, w[:3 * H], bias[:3 * H], qs, ks, cos[row_off:row_off + L], sin[row_off:row_off + L], heads)   # [L, 3H]
    r0 = rank * Ltot + row_off
    for owner in range(W):
        want = torch.cat([ref[:, reg * H + owner * hw: reg * H + (owner + 1) * hw] for reg in range(3)], dim=1)
        got = bufs[owner][r0:r0 + L].cpu()
        assert rel_l2(got, want) < 6e-3, (owner, _stats(got, want))
        assert float(bufs[owner][:r0].abs().max()) == 0 and float(bufs[owner][r0 + L:].abs().max()) == 0, "rows outside the problem were written"
    assert float(local.abs().max()) == 0
    if epi == "linear1":
        lin = (a.float() @ w[3 * H:].float().T + bias[3 * H:]).to(BF16)
        assert rel_l2(cat[row_off:row_off + L, H:].cpu(), torch.nn.functional.gelu(lin, approximate="tanh")) < 4e-3


def test_attention_sequence_parallel_row_routing(ops):
    """vcb_attention_fwd_sp: this rank's heads over all L rows; query row r goes to out_peers[r // rows] at row r % rows
    (rows = 200: the 128-row tiles straddle the owners' boundary)."""
    from oracle import flux_oracle as fo
    W, rows, heads, rank = 2, 200, 2, 1
    L, hw = W * rows, heads * 128
    qkv = _randn(L, 3 * hw, seed=17)
    ldo = W * hw + 64
    peers = [torch.zeros(rows, ldo, dtype=BF16, device="cuda") for _ in range(W)]
    ops.attention_sp(qkv.cuda(), L, heads, peers, rows, ldo, q_col=0, k_col=hw, v_col=2 * hw, out_col_offset=rank * hw)
    torch.cuda.synchronize()
    q, k, v = fo._split_heads(qkv.reshape(1, L, 3 * hw), heads)
    ref = fo.joint_attention(q, k, v, torch.ones(1, L, 64), torch.zeros(1, L, 64), torch.ones(1, L, dtype=torch.int32),
                             fo.Numerics("cuda_bf16")).reshape(L, hw)
    for owner in range(W):
        got = peers[owner].cpu()
        assert rel_l2(got[:, rank * hw:(rank + 1) * hw], ref[owner * rows:(owner + 1) * rows]) < 8e-3
        assert float(got[:, :rank * hw].abs().max()) == 0 and float(got[:, (rank + 1) * hw:].abs().max()) == 0


# ------------------------------------------------------------------------------------------------
# attention
# ------------------------------------------------------------------------------------------------
def _attn_case(ops, B, L, heads, seqlens, seed, scale=1.0):
    from oracle import flux_oracle as fo
    H = heads * 128
    qkv = _randn(B * L, 3 * H, seed=seed, scale=scale)
    out = torch.full((B * L, H), 5.0, dtype=BF16, device="cuda")
    sl = None if seqlens is None else torch.tensor(seqlens, dtype=torch.int32, device="cuda")
    ops.attention(qkv.cuda(), B, L, heads, out, q_col=0, k_col=H, v_col=2 * H, seqlens=sl)
    torch.cuda.synchronize()
    q, k, v = fo._split_heads(qkv.reshape(B, L, 3 * H), heads)
    ones, zeros = torch.ones(B, L, 64), torch.zeros(B, L, 64)
    mask = torch.ones(B, L, dtype=torch.int32)
    if seqlens is not None:
        for b, s in enumerate(seqlens):
            mask[b, s:] = 0
    ref = fo.joint_attention(q, k, v, ones, zeros, mask, fo.Numerics("cuda_bf16")).reshape(B * L, H)
    return out.cpu(), ref


@pytest.mark.parametrize("L", [128, 200, 1088, 3968])
def test_attention_full(ops, L):
    got, ref = _attn_case(ops, 1, L, 2, None, seed=L)
    # P is rounded to bf16 on both sides; O differs by fp32 summation order + final bf16 rounding
    assert rel_l2(got, ref) < 8e-3, _stats(got, ref)


def test_attention_peaked_scores_exercise_rescale(ops):
    """large-magnitude q.k -> row max jumps by >> 2^8 between tiles: exercises the O-correction path."""
    got, ref = _attn_case(ops, 1, 640, 1, None, seed=3, scale=4.0)
    assert rel_l2(got, ref) < 1e-2, _stats(got, ref)


def test_attention_ragged_batch(ops):
    """right-padded batch: masked keys, zeroed padded query rows (math.py:9-60 + pad_input)."""
    B, L, seqlens = 2, 520, [520, 301]
    got, ref = _attn_case(ops, B, L, 2, seqlens, seed=9)
    assert rel_l2(got, ref) < 8e-3, _stats(got, ref)
    assert float(got.reshape(B, L, -1)[1, 301:].abs().max()) == 0


@pytest.mark.parametrize("case", ["full", "ragged"])
def test_attention_score_bound_equals_online_softmax(ops, case):
    """vcb_attn_args.score_bound_log2: with q, k bounded like QK-RMSNorm leaves them (|q| = a*sqrt(128), |k| = b*sqrt(128))
    the fixed-reference softmax exp2(s - bound) must equal the exact online-max kernel and the oracle (shift invariance)."""
    from oracle import flux_oracle as fo
    B, L, heads = (1, 648, 2) if case == "full" else (2, 520, 2)
    seqlens = None if case == "full" else [520, 301]
    H = heads * 128
    qkv = _randn(B * L, 3 * H, seed=41).float().reshape(B * L, 3, heads, 128)
    qa, ka = 1.3, 0.9
    for i, a in ((0, qa), (1, ka)):       # unit-RMS rows times a scale, as after RMSNorm * scale (layers.py:63-84)
        qkv[:, i] = a * qkv[:, i] / qkv[:, i].pow(2).mean(-1, keepdim=True).sqrt()
    qkv = qkv.reshape(B * L, 3 * H).to(BF16)
    bound = qa * ka * math.sqrt(128.0) * math.log2(math.e) * 1.03
    sl = None if seqlens is None else torch.tensor(seqlens, dtype=torch.int32, device="cuda")
    outs = []
    for sb in (0.0, bound):
        out = torch.full((B * L, H), 5.0, dtype=BF16, device="cuda")
        ops.attention(qkv.cuda(), B, L, heads, out, q_col=0, k_col=H, v_col=2 * H, seqlens=sl, score_bound_log2=sb)
        torch.cuda.synchronize()
        outs.append(out.cpu())
    q, k, v = fo._split_heads(qkv.reshape(B, L, 3 * H), heads)
    mask = torch.ones(B, L, dtype=torch.int32)
    if seqlens is not None:
        for b, n in enumerate(seqlens):
            mask[b, n:] = 0
    ref = fo.joint_attention(q, k, v, torch.ones(B, L, 64), torch.zeros(B, L, 64), mask, fo.Numerics("cuda_bf16")).reshape(B * L, H)
    assert rel_l2(outs[1], ref) < 8e-3, _stats(outs[1], ref)
    assert rel_l2(outs[1], outs[0]) < 5e-3, _stats(outs[1], outs[0])
    if seqlens is not None:
        assert float(outs[1].reshape(B, L, H)[1, 301:].abs().max()) == 0, "padded query rows must be zero"
    with pytest.raises(Exception, match="score_bound_log2"):
        ops.attention(qkv.cuda(), B, L, heads, torch.empty_like(outs[0]).cuda(), q_col=0, k_col=H, v_col=2 * H, score_bound_log2=80.0)


def test_attention_strided_output_columns(ops):
    """writes into columns [0, H) of the [L, H + mlp] linear2 input of a single block."""
    from oracle import flux_oracle as fo
    B, L, heads = 1, 256, 2
    H = heads * 128
    qkv = _randn(L, 3 * H, seed=4)
    cat = torch.zeros(L, H + 512, dtype=BF16, device="cuda")
    ops.attention(qkv.cuda(), B, L, heads, cat, q_col=0, k_col=H, v_col=2 * H)
    q, k, v = fo._split_heads(qkv.reshape(B, L, 3 * H), heads)
    ref = fo.joint_attention(q, k, v, torch.ones(B, L, 64), torch.zeros(B, L, 64), torch.ones(B, L, dtype=torch.int32),
                             fo.Numerics("cuda_bf16")).reshape(L, H)
    assert rel_l2(cat[:, :H].cpu(), ref) < 8e-3, _stats(cat[:, :H], ref)
    assert float(cat[:, H:].abs().max()) == 0


# ------------------------------------------------------------------------------------------------
# elementwise
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("H", [256, 3072])
def test_ln_modulate(ops, H):
    from oracle import flux_oracle as fo
    B, Lb = 2, 77
    x = _randn(B * Lb, H, seed=1, scale=2.0)
    shift, scale = _randn(B, H, seed=2, scale=0.5), _randn(B, H, seed=3, scale=0.5)
    out = torch.empty(B * Lb, H, dtype=BF16, device="cuda")
    ops.ln_modulate(x.cuda(), shift.cuda(), scale.cuda(), out, rows_per_batch=Lb)
    ref = fo._modulate(x.reshape(B, Lb, H), shift[:, None], scale[:, None], fo.Numerics("cuda_bf16")).to(BF16)
    # identical rounding points; fp32 statistics differ in summation order only
    assert rel_l2(out.cpu(), ref.reshape(B * Lb, H)) < 2e-3, _stats(out, ref.reshape(B * Lb, H))


def test_ln_modulate_grouped_two_streams_one_launch(ops):
    """img and txt streams of a double block (their own shift / scale, rows interleaved per sample in the joint buffer) in ONE
    launch must equal two separate launches bit for bit."""
    B, Lt, Li, H = 2, 24, 83, 512
    L = Lt + Li
    x = _randn(B * L, H, seed=61, scale=2.0).cuda()
    mods = [_randn(B, 6 * H, seed=62 + s, scale=0.5).cuda() for s in range(2)]       # [B, 6H] rows: shift at col 0, scale at col H
    ref = torch.zeros_like(x)
    for s, (rows, off) in enumerate(((Li, Lt), (Lt, 0))):
        ops.ln_modulate(x[off:], mods[s][:, 0:H], mods[s][:, H:2 * H], ref[off:], rows_per_batch=rows, mod_stride=6 * H,
                        rows=B * rows, batch_rows=L)
    got = torch.zeros_like(x)
    ops.ln_modulate_grouped(x, got, [(Lt, B * Li, Li, mods[0][:, 0:H], mods[0][:, H:2 * H]),
                                     (0, B * Lt, Lt, mods[1][:, 0:H], mods[1][:, H:2 * H])], H, L, 6 * H)
    torch.cuda.synchronize()
    assert torch.equal(got, ref)
    assert float(ref.abs().max()) > 0


def test_timestep_embedding_silu_add3(ops):
    from oracle import flux_oracle as fo
    t = torch.tensor([1.0, 0.76096, 0.25, 0.0])
    g = torch.full((4,), 30.0, dtype=BF16)
    freqs = torch.exp(-math.log(10000) * torch.arange(0, 128, dtype=torch.float32) / 128)
    for tin, ref in ((1000.0 * t, fo.timestep_embedding(t).to(BF16)), ((1000.0 * g).float(), fo.timestep_embedding(g))):
        out = torch.empty(4, 256, dtype=BF16, device="cuda")
        ops.timestep_embedding(tin.cuda(), freqs.cuda(), out)
        assert (out.cpu().float() - ref.float()).abs().max() < 1.6e-2, _stats(out, ref)   # 1-2 bf16 ulp at |x|<=1
    x = _randn(4, 512, seed=1, scale=3)
    y = torch.empty_like(x, device="cuda")
    ops.silu(x.cuda(), y)
    assert rel_l2(y.cpu(), torch.nn.functional.silu(x)) < 3e-3
    a, b, c = _randn(6, 512, seed=2), _randn(2, 512, seed=3), _randn(2, 512, seed=4)
    o = torch.empty(6, 512, dtype=BF16, device="cuda")
    ops.add3(a.cuda(), b.cuda(), c.cuda(), o)
    ref = (a.reshape(3, 2, 512) + b[None]) + c[None]
    assert torch.equal(o.cpu(), ref.reshape(6, 512))


def test_rope_table_and_euler(ops):
    from oracle import flux_oracle as fo
    ids = torch.zeros(300, 3)
    ids[:, 0] = torch.arange(300) % 3 + 1
    ids[:, 1] = torch.arange(300) // 24
    ids[:, 2] = torch.arange(300) % 72
    out = torch.empty(64, 300, 2, dtype=torch.float32, device="cuda")
    ops.rope_table(ids.cuda(), [16, 56, 56], 10000, out)
    cos, sin = fo.rope_table(ids[None], [16, 56, 56], 10000)
    assert (out[..., 0].cpu().T - cos[0]).abs().max() < 1e-6 and (out[..., 1].cpu().T - sin[0]).abs().max() < 1e-6
    x, v = _randn(500, 64, seed=1), _randn(500, 64, seed=2)
    dt = torch.tensor(1.0 / 29)                                  # 0-dim fp32 like torchdiffeq's dt
    ref = x + dt * (-v)                                          # torch promotion -> bf16(x + bf16(bf16(dt)*f))
    xn = torch.empty(500, 64, dtype=BF16, device="cuda")
    inp = torch.zeros(500, 384, dtype=BF16, device="cuda")
    ops.euler_update(x.cuda(), v.cuda(), float(dt.to(BF16)), xn, inp)
    assert torch.equal(xn.cpu(), ref), _stats(xn, ref)
    assert torch.equal(inp[:, :64].cpu(), ref) and float(inp[:, 64:].abs().max()) == 0


def test_gemm_streamk_enabled_subprocess():
    """The stream-K tail is off by default (DESIGN.md section 5); run it explicitly in a child process (the switch is read once
    per process) on a shape whose last wave is half empty, grouped and plain, and compare with fp32 matmul."""
    import os
    import subprocess
    import sys
    code = r"""
import math, sys, torch
sys.path.insert(0, %r)
from visualcloze_b200 import ops
g = torch.Generator().manual_seed(0)
M, N, K = 3968, 3072, 4096
a = torch.randn(M, K, generator=g).bfloat16(); w = (torch.randn(N, K, generator=g) / math.sqrt(K)).bfloat16()
bias = torch.randn(N, generator=g)
out = torch.empty(M, N, dtype=torch.bfloat16, device="cuda")
ops.gemm(a.cuda(), w.cuda(), bias.cuda(), out, cta_group=2, block_n=256)
torch.cuda.synchronize()
ref = (a.float() @ w.float().T + bias).bfloat16().float()
err = float((out.float().cpu() - ref).norm() / ref.norm())
assert err < 3e-3, err
# fewer tiles than CTA pairs (36 on 74): every pair gets an equal K range of the few tiles
M = 600
a = torch.randn(M, 8192, generator=g).bfloat16(); w = (torch.randn(N, 8192, generator=g) / math.sqrt(8192)).bfloat16()
out = torch.empty(M, N, dtype=torch.bfloat16, device="cuda")
for cg in (1, 2):
    ops.gemm(a.cuda(), w.cuda(), bias.cuda(), out, cta_group=cg, block_n=256)
    torch.cuda.synchronize()
    ref = (a.float() @ w.float().T + bias).bfloat16().float()
    err2 = float((out.float().cpu() - ref).norm() / ref.norm())
    assert err2 < 3e-3, (cg, err2)
print("streamk ok", err)
""" % os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, "-c", code], env=dict(os.environ, VCB_STREAMK="1"), capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "streamk ok" in r.stdout, r.stdout + r.stderr


# ------------------------------------------------------------------------------------------------
# attention: persistent schedule (attn4) -- units cut at a CTA's share boundary are folded from fp32 partials
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("shape", [(1, 2, 128), (1, 2, 200), (1, 2, 1088), (1, 3, 1500), (2, 2, 520), (1, 1, 640), (1, 2, 3968)])
@pytest.mark.parametrize("bounded", [False, True])
def test_attention_persistent_schedule_matches_per_pair_and_oracle(ops, shape, bounded):
    """vcb_attn_args.schedule: PERSISTENT (one CTA per SM, equal shares, 1..4 pieces per cut unit) vs PER_PAIR vs the oracle, for
    both softmax variants; shapes chosen so shares cut units mid-way, across heads, and (L = 200, 1500, 520) at ragged tile edges."""
    from oracle import flux_oracle as fo
    B, heads, L = shape
    H = heads * 128
    qkv = _randn(B * L, 3 * H, seed=L + heads).float().reshape(B * L, 3, heads, 128)
    qa, ka = 1.3, 0.9
    for i, a in ((0, qa), (1, ka)):
        qkv[:, i] = a * qkv[:, i] / qkv[:, i].pow(2).mean(-1, keepdim=True).sqrt()
    qkv = qkv.reshape(B * L, 3 * H).to(BF16)
    sb = qa * ka * math.sqrt(128.0) * math.log2(math.e) * 1.03 if bounded else 0.0
    outs = {}
    for sched in (1, 2):
        out = torch.full((B * L, H), 5.0, dtype=BF16, device="cuda")
        ops.attention(qkv.cuda(), B, L, heads, out, q_col=0, k_col=H, v_col=2 * H, score_bound_log2=sb, schedule=sched)
        torch.cuda.synchronize()
        outs[sched] = out.cpu()
    q, k, v = fo._split_heads(qkv.reshape(B, L, 3 * H), heads)
    ref = fo.joint_attention(q, k, v, torch.ones(B, L, 64), torch.zeros(B, L, 64), torch.ones(B, L, dtype=torch.int32),
                             fo.Numerics("cuda_bf16")).reshape(B * L, H)
    assert rel_l2(outs[2], ref) < 8e-3, _stats(outs[2], ref)
    assert rel_l2(outs[2], outs[1]) < 5e-3, _stats(outs[2], outs[1])


def test_attention_persistent_back_to_back_launches_reuse_the_workspace(ops):
    """the per-stream (O, l, m) slots and flags are reused by every launch (epoch-tagged): 20 launches in a row must all agree"""
    B, heads, L = 1, 4, 2000
    H = heads * 128
    qkv = _randn(B * L, 3 * H, seed=77).cuda()
    outs = []
    for i in range(20):
        out = torch.empty(B * L, H, dtype=BF16, device="cuda")
        ops.attention(qkv, B, L, heads, out, q_col=0, k_col=H, v_col=2 * H, schedule=2)
        outs.append(out)
    torch.cuda.synchronize()
    for o in outs[1:]:
        assert torch.equal(o, outs[0])


def test_attention_persistent_rejects_padded_batches(ops):
    qkv = _randn(2 * 256, 3 * 256, seed=1).cuda()
    sl = torch.tensor([256, 100], dtype=torch.int32, device="cuda")
    with pytest.raises(Exception, match="persistent"):
        ops.attention(qkv, 2, 256, 2, torch.empty(512, 256, dtype=BF16, device="cuda"), q_col=0, k_col=256, v_col=512, seqlens=sl, schedule=2)


# ------------------------------------------------------------------------------------------------
# LayerNorm statistics produced by the GATE_RES epilogue (row_stats) and consumed by vcb_ln_modulate_stats
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cfg", [(256, 2), (256, 1), (128, 1), (128, 2), (0, 0)])
def test_gate_res_row_stats_and_stats_layernorm(ops, cfg):
    """x += gate * (a w^T + b) with row_stats: per row and per 64 columns (sum, sum of squares) of the bf16 values written; the
    LayerNorm fed with them must equal the two-pass LayerNorm kernel on the same x (statistics differ only in fp32 summation
    order) -- grouped img + txt problems, row-mapped output like a DoubleStreamBlock's proj launch."""
    bn, cg = cfg
    g = torch.Generator().manual_seed(13)
    K, N, Li, Lt = 512, 768, 450, 70
    L = Li + Lt
    a = torch.randn(L, K, generator=g).to(BF16).cuda()
    x0 = torch.randn(L, N, generator=g).to(BF16)
    x = x0.clone().cuda()
    stats = torch.full((L, N // 64, 2), -7.0, dtype=torch.float32, device="cuda")
    probs = []
    for off, rows in ((Lt, Li), (0, Lt)):
        w = (torch.randn(N, K, generator=g) / math.sqrt(K)).to(BF16).cuda()
        bias = torch.randn(N, generator=g).cuda()
        gate = (0.5 * torch.randn(1, N, generator=g)).to(BF16).cuda()
        probs.append(dict(a=a[off:off + rows], w=w, bias=bias, out=x, epilogue=ops.EPI_GATE_RES, gate=gate, res=x, rows_per_batch=rows,
                          out_batch_rows=L, out_row_offset=off, row_stats=stats, block_n=bn, cta_group=cg))
    ops.gemm_grouped(probs[0], probs[1])
    torch.cuda.synchronize()
    xf = x.float().reshape(L, N // 64, 64)
    ref = torch.stack((xf.sum(-1), (xf * xf).sum(-1)), dim=-1)
    assert torch.allclose(stats, ref, rtol=2e-5, atol=2e-4), float((stats - ref).abs().max())
    shift = (0.2 * torch.randn(1, N, generator=g)).to(BF16).cuda()
    scale = (0.3 * torch.randn(1, N, generator=g)).to(BF16).cuda()
    y_two = torch.empty(L, N, dtype=BF16, device="cuda")
    y_st = torch.empty(L, N, dtype=BF16, device="cuda")
    ops.ln_modulate(x, shift, scale, y_two, rows_per_batch=L)
    ops.ln_modulate_stats(x, shift, scale, y_st, stats, rows_per_batch=L)
    torch.cuda.synchronize()
    assert rel_l2(y_st.cpu(), y_two.cpu()) < 2e-3
    assert float((y_st.float() - y_two.float()).abs().max()) <= 0.0625       # a few bf16 ulps at |y| <= ~8 where the fp32 statistics round differently


def test_row_stats_rejected_where_it_cannot_work(ops):
    a = torch.zeros(128, 256, dtype=BF16, device="cuda")
    w = torch.zeros(128, 256, dtype=BF16, device="cuda")
    out = torch.zeros(128, 128, dtype=BF16, device="cuda")
    st = torch.zeros(128, 2, 2, device="cuda")
    with pytest.raises(Exception, match="row_stats"):
        ops.gemm(a, w, None, out, row_stats=st)                                  # not the GATE_RES epilogue
    with pytest.raises(Exception, match="row_stats"):
        ops.gemm(a, w, None, out, epilogue=ops.EPI_GATE_RES, res=out, gate=torch.zeros(1, 128, dtype=BF16, device="cuda"), row_stats=st, block_n=192)


@pytest.mark.parametrize("raster", ["0", "1"])
def test_gemm_tile_raster_forced_subprocess(raster):
    """GemmParams.n_fastest is chosen per shape (A bigger than B -> N-fastest); force each raster in a child process (the switch
    is read once per process) over plain, batched, grouped and head-structured launches and compare with fp32 matmul."""
    import os
    import subprocess
    import sys
    code = r"""
import math, sys, torch
sys.path.insert(0, %r)
from visualcloze_b200 import ops
BF16 = torch.bfloat16
g = torch.Generator().manual_seed(1)
def rel(a, b): return float((a.double() - b.double()).norm() / b.double().norm())
for (M, N, K) in ((1000, 512, 384), (300, 1536, 512), (3968, 3072, 1024)):
    a = torch.randn(M, K, generator=g).to(BF16); w = (torch.randn(N, K, generator=g) / math.sqrt(K)).to(BF16); b = torch.randn(N, generator=g)
    out = torch.empty(M, N, dtype=BF16, device="cuda")
    ops.gemm(a.cuda(), w.cuda(), b.cuda(), out)
    assert rel(out.cpu(), (a.float() @ w.float().T + b).to(BF16)) < 4e-3, (M, N, K)
# batched rows with a row-mapped output (two samples of 260 rows inside 300-row slots)
B, R, S, N, K = 2, 260, 300, 384, 256
a = torch.randn(B * R, K, generator=g).to(BF16); w = (torch.randn(N, K, generator=g) / math.sqrt(K)).to(BF16); bias = torch.randn(N, generator=g)
out = torch.zeros(B * S, N, dtype=BF16, device="cuda")
ops.gemm(a.cuda(), w.cuda(), bias.cuda(), out, rows_per_batch=R, out_batch_rows=S, out_row_offset=20)
ref = (a.float() @ w.float().T + bias).to(BF16).reshape(B, R, N)
got = out.cpu().reshape(B, S, N)
assert rel(got[:, 20:20 + R], ref) < 4e-3 and float(got[:, :20].abs().max()) == 0 and float(got[:, 20 + R:].abs().max()) == 0
# grouped img + txt problems with the gated-residual epilogue
K, N, Li, Lt = 512, 256, 900, 130
L = Li + Lt
a = torch.randn(L, K, generator=g).to(BF16).cuda(); x0 = torch.randn(L, N, generator=g).to(BF16); x = x0.clone().cuda()
probs, refs = [], []
for off, rows in ((Lt, Li), (0, Lt)):
    w = (torch.randn(N, K, generator=g) / math.sqrt(K)).to(BF16); bias = torch.randn(N, generator=g); gate = (0.5 * torch.randn(1, N, generator=g)).to(BF16)
    probs.append(dict(a=a[off:off + rows], w=w.cuda(), bias=bias.cuda(), out=x, epilogue=ops.EPI_GATE_RES, gate=gate.cuda(), res=x, rows_per_batch=rows,
                      out_batch_rows=L, out_row_offset=off))
    lin = (a[off:off + rows].cpu().float() @ w.float().T + bias).to(BF16)
    refs.append((off, rows, (x0[off:off + rows].float() + (gate.float() * lin.float()).to(BF16).float()).to(BF16)))
ops.gemm_grouped(probs[0], probs[1])
torch.cuda.synchronize()
for off, rows, ref in refs:
    assert rel(x[off:off + rows].cpu(), ref) < 4e-3
print("raster ok")
""" % os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, "-c", code], env=dict(os.environ, VCB_GEMM_RASTER=raster), capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "raster ok" in r.stdout, r.stdout[-2000:] + r.stderr[-2000:]
