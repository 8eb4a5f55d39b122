"""Unmerged LoRA on the H100: the GEMM's LoRA k-tail against fp32 torch, the model in unmerged mode against the restated
oracle (which is itself unmerged, lora.py:92-98) and against the merged mode, copy-free packing, adapter switching, and the
full FLUX geometry against the reference.

Tolerances: kernel level as the bf16 GEMM tests of test_kernels_gpu.py (BIAS 3e-3, GELU / GATE_RES 4e-3, QKV / LINEAR1 6e-3);
model level as test_flux_gpu.py (forward 2e-2, trajectory 5e-2); unmerged vs merged 1e-2 (the two differ by where the update
is rounded: bf16(W + sBA) once per weight vs s * (x A^T) rounded to bf16 per call)."""
import dataclasses
import math
import os
import tempfile

import pytest
import torch

from conftest import GOLDEN, REPO, rel_l2

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


def _operands(M, N, K, r, seed=0):
    a, w = _randn(M, K, seed=seed + 1), _randn(N, K, seed=seed + 2, scale=1 / math.sqrt(K))
    t, lb = _randn(M, r, seed=seed + 3), _randn(N, r, seed=seed + 4, scale=1 / math.sqrt(r))
    bias = _randn(N, seed=seed + 5, dtype=torch.float32, scale=0.1)
    acc = a.float() @ w.float().T + t.float() @ lb.float().T
    return a, w, t, lb, bias, acc


def _qkv_ref(lin, qs, ks, cos, sin, heads):
    from oracle import flux_oracle as fo
    L = lin.shape[0]
    q, k, v = fo._split_heads(lin[None], heads)
    q = fo.apply_rope(fo.rms_norm(q, qs), cos[None], sin[None])
    k = fo.apply_rope(fo.rms_norm(k, ks), cos[None], sin[None])
    return torch.cat([x.permute(0, 2, 1, 3).reshape(L, -1) for x in (q, k, v)], dim=-1)


def _rope(rows, seed):
    ang = _randn(rows, 64, seed=seed, dtype=torch.float32) * 3
    cos, sin = torch.cos(ang), torch.sin(ang)
    return cos, sin, torch.stack([cos, sin], -1).permute(1, 0, 2).contiguous()


# ------------------------------------------------------------------------------------------------
# kernel level
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("rank", [256, 64, 72])
@pytest.mark.parametrize("cta_group", [1, 2])
@pytest.mark.parametrize("block_n", [128, 256])
def test_ktail_bias(ops, rank, cta_group, block_n):
    M, N, K = 520, 768, 384
    a, w, t, lb, bias, acc = _operands(M, N, K, rank)
    out = torch.full((M, N), 7.0, dtype=BF16, device="cuda")
    ops.gemm(a.cuda(), w.cuda(), bias.cuda(), out, lora_t=t.cuda(), lora_b=lb.cuda(), block_n=block_n, cta_group=cta_group)
    ref = (acc + bias).to(BF16)
    assert rel_l2(out.cpu(), ref) < 3e-3


@pytest.mark.parametrize("cta_group", [1, 2])
def test_ktail_gelu(ops, cta_group):
    M, N, K, r = 520, 1024, 256, 72
    a, w, t, lb, bias, acc = _operands(M, N, K, r, seed=10)
    out = torch.empty(M, N, dtype=BF16, device="cuda")
    ops.gemm(a.cuda(), w.cuda(), bias.cuda(), out, epilogue=ops.EPI_BIAS_GELU, lora_t=t.cuda(), lora_b=lb.cuda(), cta_group=cta_group)
    ref = torch.nn.functional.gelu((acc + bias).to(BF16), approximate="tanh")
    assert rel_l2(out.cpu(), ref) < 4e-3


@pytest.mark.parametrize("cta_group", [1, 2])
def test_ktail_gate_residual_row_stats_batched_row_offset(ops, cta_group):
    """Two samples of a joint [B, L, *] buffer written at a row offset (the img stream), in-place gated residual, with the
    LayerNorm statistics the epilogue leaves behind; T addressed like A (its own row stride and batch stride)."""
    B, Lt, Li, H, K, r = 2, 40, 300, 512, 256, 64
    L = Li + Lt
    a = _randn(B * L, K, seed=20)
    tbuf = _randn(B * L, r + 8, seed=21)                              # row stride r + 8: T is a column window of a wider buffer
    w, lb = _randn(H, K, seed=22, scale=1 / math.sqrt(K)), _randn(H, r, seed=23, scale=1 / math.sqrt(r))
    bias = _randn(H, seed=24, dtype=torch.float32, scale=0.1)
    gate, x = _randn(B, H, seed=25), _randn(B * L, H, seed=26)
    xg, ag, tg = x.cuda().clone(), a.cuda(), tbuf.cuda()
    stats = torch.full((B * L, H // 64, 2), 1e9, dtype=torch.float32, device="cuda")
    ops.gemm(ag[Lt:], w.cuda(), bias.cuda(), xg, epilogue=ops.EPI_GATE_RES, m=B * Li, rows_per_batch=Li, out_batch_rows=L,
             out_row_offset=Lt, a_batch_stride=L * K, gate=gate.cuda(), res=xg, cta_group=cta_group, block_n=256, row_stats=stats,
             lora_t=tg[Lt:, :r], lora_b=lb.cuda(), lora_t_batch_stride=L * (r + 8))
    a3, t3 = a.reshape(B, L, K)[:, Lt:], tbuf.reshape(B, L, r + 8)[:, Lt:, :r]
    lin = (a3.float() @ w.float().T + t3.float() @ lb.float().T + bias).to(BF16)
    ref = x.reshape(B, L, H).clone()
    ref[:, Lt:] = x.reshape(B, L, H)[:, Lt:] + gate[:, None, :] * lin
    got = xg.cpu()
    assert rel_l2(got, ref.reshape(B * L, H)) < 4e-3
    assert torch.equal(got.reshape(B, L, H)[:, :Lt], x.reshape(B, L, H)[:, :Lt]), "txt rows untouched"
    # statistics of the stored bf16 values, per 64 columns, at the mapped output rows only
    st = stats.cpu().reshape(B, L, H // 64, 2)
    g64 = got.reshape(B, L, H // 64, 64).float()[:, Lt:]
    assert torch.allclose(st[:, Lt:, :, 0], g64.sum(-1), rtol=1e-4, atol=1e-3)
    assert torch.allclose(st[:, Lt:, :, 1], g64.pow(2).sum(-1), rtol=1e-4, atol=1e-3)
    assert float(st[:, :Lt].min()) == 1e9


@pytest.mark.parametrize("cta_group", [1, 2])
@pytest.mark.parametrize("block_n", [128, 256])
def test_ktail_qkv(ops, block_n, cta_group):
    L, H, heads, K, r, row_off, Ltot = 200, 256, 2, 256, 72, 24, 256
    a, w, t, lb, bias, acc = _operands(L, 3 * H, K, r, seed=30)
    qs, ks = (1 + 0.1 * _randn(128, seed=34, dtype=torch.float32)).to(BF16), (1 + 0.1 * _randn(128, seed=35, dtype=torch.float32)).to(BF16)
    cos, sin, rope = _rope(Ltot, 36)
    out = torch.zeros(Ltot, 3 * H, dtype=BF16, device="cuda")
    ops.gemm(a.cuda(), w.cuda(), bias.cuda(), out, epilogue=ops.EPI_QKV, hidden=H, q_scale=qs.cuda(), k_scale=ks.cuda(),
             rope=rope.cuda(), rows_per_batch=L, out_batch_rows=Ltot, out_row_offset=row_off, block_n=block_n, cta_group=cta_group,
             lora_t=t.cuda(), lora_b=lb.cuda())
    ref = _qkv_ref((acc + bias).to(BF16), qs, ks, cos[row_off:row_off + L], sin[row_off:row_off + L], heads)
    assert rel_l2(out[row_off:row_off + L].cpu(), ref) < 6e-3


@pytest.mark.parametrize("cta_group", [1, 2])
def test_ktail_linear1(ops, cta_group):
    L, H, heads, mlp, r = 160, 256, 2, 512, 64
    a, w, t, lb, bias, acc = _operands(L, 3 * H + mlp, H, r, seed=40)
    qs, ks = (1 + 0.1 * _randn(128, seed=44, dtype=torch.float32)).to(BF16), (1 + 0.1 * _randn(128, seed=45, dtype=torch.float32)).to(BF16)
    cos, sin, rope = _rope(L, 46)
    qkv = torch.zeros(L, 3 * H, dtype=BF16, device="cuda")
    cat = torch.zeros(L, H + mlp, dtype=BF16, device="cuda")
    ops.gemm(a.cuda(), w.cuda(), bias.cuda(), qkv, epilogue=ops.EPI_LINEAR1, hidden=H, q_scale=qs.cuda(), k_scale=ks.cuda(),
             rope=rope.cuda(), out2=cat, out2_col_offset=H, cta_group=cta_group, lora_t=t.cuda(), lora_b=lb.cuda())
    lin = (acc + bias).to(BF16)
    assert rel_l2(qkv.cpu(), _qkv_ref(lin[:, :3 * H], qs, ks, cos, sin, heads)) < 6e-3
    assert rel_l2(cat[:, H:].cpu(), torch.nn.functional.gelu(lin[:, 3 * H:], approximate="tanh")) < 4e-3


@pytest.mark.parametrize("cta_group", [0, 1, 2])
def test_ktail_grouped_two_streams(ops, cta_group):
    """img + txt streams in ONE launch, each with its own T rows and lora_b (same rank)."""
    B, Li, Lt, H, K, r = 2, 300, 40, 512, 256, 72
    L = Li + Lt
    attn, tj, x = _randn(B * L, K, seed=50), _randn(B * L, r, seed=51), _randn(B * L, H, seed=52)
    w = [_randn(H, K, seed=53 + s, scale=1 / math.sqrt(K)) for s in range(2)]
    lb = [_randn(H, r, seed=55 + s, scale=1 / math.sqrt(r)) for s in range(2)]
    bias = [_randn(H, seed=57 + s, dtype=torch.float32, scale=0.1) for s in range(2)]
    gate = [_randn(B, H, seed=59 + s) for s in range(2)]
    xg, ag, tg = x.cuda().clone(), attn.cuda(), tj.cuda()
    probs = []
    for s, (rows, off) in enumerate(((Li, Lt), (Lt, 0))):
        probs.append(dict(a=ag[off:], w=w[s].cuda(), bias=bias[s].cuda(), out=xg, epilogue=ops.EPI_GATE_RES, m=B * rows,
                          rows_per_batch=rows, out_batch_rows=L, out_row_offset=off, a_batch_stride=L * K, gate=gate[s].cuda(),
                          res=xg, cta_group=cta_group, lora_t=tg[off:], lora_b=lb[s].cuda(), lora_t_batch_stride=L * r))
    ops.gemm_grouped(probs[0], probs[1])
    ref = x.reshape(B, L, H).clone()
    a3, t3 = attn.reshape(B, L, K), tj.reshape(B, L, r)
    for s, (rows, off) in enumerate(((Li, Lt), (Lt, 0))):
        lin = (a3[:, off:off + rows].float() @ w[s].float().T + t3[:, off:off + rows].float() @ lb[s].float().T + bias[s]).to(BF16)
        ref[:, off:off + rows] = x.reshape(B, L, H)[:, off:off + rows] + gate[s][:, None, :] * lin
    assert rel_l2(xg.cpu(), ref.reshape(B * L, H)) < 4e-3


def test_ktail_grouped_rejects_different_ranks(ops):
    from visualcloze_b200._lib import VcbError
    a, w, t, lb, bias, _ = _operands(256, 256, 256, 64)
    t2, lb2 = _randn(256, 72, seed=9), _randn(256, 72, seed=8)
    out = torch.empty(256, 256, dtype=BF16, device="cuda")
    p0 = dict(a=a.cuda(), w=w.cuda(), bias=None, out=out, lora_t=t.cuda(), lora_b=lb.cuda())
    with pytest.raises(VcbError, match="rank"):
        ops.gemm_grouped(p0, dict(p0, lora_t=t2.cuda(), lora_b=lb2.cuda()))
    with pytest.raises(VcbError, match="lora_rank"):
        ops.gemm(a.cuda(), w.cuda(), None, out, lora_t=t[:, :60].cuda(), lora_b=lb[:, :60].contiguous().cuda())


def test_ktail_streamk_tail_subprocess():
    """The stream-K tail cuts the k range of the partial last wave, LoRA k-blocks included: forced on in a child process (the
    switch is read once per process), few tiles and a long K, both cta groups, a plain and a grouped launch."""
    import subprocess
    import sys
    code = r"""
import math, sys, torch
sys.path.insert(0, %r)
from visualcloze_b200 import ops
g = torch.Generator().manual_seed(0)
M, N, K, r = 600, 3072, 8192, 256
a = torch.randn(M, K, generator=g).bfloat16(); w = (torch.randn(N, K, generator=g) / math.sqrt(K)).bfloat16()
t = torch.randn(M, r, generator=g).bfloat16(); lb = (torch.randn(N, r, generator=g) / math.sqrt(r)).bfloat16()
bias = torch.randn(N, generator=g)
ref = (a.float() @ w.float().T + t.float() @ lb.float().T + bias).bfloat16().float()
for cg in (1, 2):
    out = torch.empty(M, N, dtype=torch.bfloat16, device="cuda")
    ops.gemm(a.cuda(), w.cuda(), bias.cuda(), out, cta_group=cg, block_n=256, lora_t=t.cuda(), lora_b=lb.cuda())
    torch.cuda.synchronize()
    err = float((out.float().cpu() - ref).norm() / ref.norm())
    assert err < 3e-3, (cg, err)
    outs = [torch.empty(M // 2, N, dtype=torch.bfloat16, device="cuda") for _ in range(2)]
    p = [dict(a=a[h * M // 2:(h + 1) * M // 2].cuda(), w=w.cuda(), bias=bias.cuda(), out=outs[h], cta_group=cg, block_n=256,
              lora_t=t[h * M // 2:(h + 1) * M // 2].cuda(), lora_b=lb.cuda()) for h in range(2)]
    ops.gemm_grouped(p[0], p[1])
    torch.cuda.synchronize()
    err2 = float((torch.cat(outs).float().cpu() - ref).norm() / ref.norm())
    assert err2 < 3e-3, (cg, err2)
print("streamk lora ok")
""" % REPO
    r = subprocess.run([sys.executable, "-c", code], env=dict(os.environ, VCB_STREAMK="1"), capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "streamk lora ok" in r.stdout, r.stdout + r.stderr


def _ulp_bf16(x):
    e = torch.floor(torch.log2(x.float().abs().clamp_min(1e-30)))
    return torch.pow(2.0, e - 7)


@pytest.mark.parametrize("cta_group", [1, 2])
def test_zero_lora_b_matches_the_tail_free_gemm(ops, cta_group):
    """A zero lora_b adds exact zeros to the accumulator: bitwise the tail-free GEMM where no stream-K split is taken (a few
    tiles), within one bf16 ulp on a multi-wave shape (where the split points may move with the longer k range)."""
    for (M, N, K), exact in (((256, 256, 512), True), ((3000, 3072, 512), False)):
        a, w, t, lb, bias, _ = _operands(M, N, K, 64, seed=60)
        ag, wg, bg = a.cuda(), w.cuda(), bias.cuda()
        base = torch.empty(M, N, dtype=BF16, device="cuda")
        tail = torch.empty(M, N, dtype=BF16, device="cuda")
        ops.gemm(ag, wg, bg, base, block_n=256, cta_group=cta_group)
        ops.gemm(ag, wg, bg, tail, block_n=256, cta_group=cta_group, lora_t=t.cuda(), lora_b=torch.zeros_like(lb).cuda())
        if exact:
            assert torch.equal(base, tail)
        d = (base.float() - tail.float()).abs().cpu()
        assert bool((d <= _ulp_bf16(base.cpu()) + 1e-30).all()), float(d.max())


def test_alpha_scales_the_down_projection(ops):
    M, N, K = 700, 256, 3072
    a, w = _randn(M, K, seed=70), _randn(N, K, seed=71, scale=1 / math.sqrt(K))
    for alpha in (0.5, -1.75):
        out = torch.empty(M, N, dtype=BF16, device="cuda")
        ops.gemm(a.cuda(), w.cuda(), None, out, alpha=alpha)
        ref = (alpha * (a.float() @ w.float().T)).to(BF16)
        assert rel_l2(out.cpu(), ref) < 3e-3
    # 0 and 1 both mean "no scaling": bitwise the plain GEMM
    outs = []
    for alpha in (0.0, 1.0):
        outs.append(torch.empty(M, N, dtype=BF16, device="cuda"))
        ops.gemm(a.cuda(), w.cuda(), None, outs[-1], alpha=alpha)
    assert torch.equal(outs[0], outs[1])


# ------------------------------------------------------------------------------------------------
# model level
# ------------------------------------------------------------------------------------------------
def _load(name):
    return torch.load(os.path.join(GOLDEN, name), weights_only=False)


def _cuda(d):
    return {k: (v.cuda() if torch.is_tensor(v) else v) for k, v in d.items()}


def _build(cfg_dict, seed, mode="unmerged"):
    import visualcloze_b200.model as m
    from oracle import flux_oracle as fo
    cfg = fo.FluxConfig(**cfg_dict)
    params = fo.make_params(cfg, seed=seed)
    fp = m.FluxParams(**{k: v for k, v in cfg_dict.items() if k not in ("lora_rank", "lora_scale")})
    with torch.device("cuda"):
        model = m.FluxLoraWrapper(lora_rank=cfg.lora_rank, params=fp)
    model.load_state_dict({k: v.cuda() for k, v in params.items()}, strict=True)
    model.set_lora_mode(mode)
    return cfg, params, model


def _full_width_case(depth=1, depth_single=1, rank=32):
    cfg_dict = dict(in_channels=384, out_channels=64, vec_in_dim=768, context_in_dim=4096, hidden_size=3072, mlp_ratio=4.0,
                    num_heads=24, depth=depth, depth_single_blocks=depth_single, axes_dim=[16, 56, 56], theta=10_000, qkv_bias=True,
                    guidance_embed=True, lora_rank=rank)
    g = torch.Generator().manual_seed(5)
    B, Lt = 1, 96
    ids = []
    for j, (h, w) in enumerate([(6, 18), (6, 18)]):
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
    return cfg_dict, inp


@pytest.mark.parametrize("tag", ["b1", "b2r", "full_width"])
def test_unmerged_forward_vs_oracle_and_merged(ops, tag):
    from oracle import flux_oracle as fo
    if tag == "full_width":
        cfg_dict, inp = _full_width_case()
        seed = 21
    else:
        g = _load(f"flux_small_{tag}.pt")
        cfg_dict, inp, seed = g["cfg"], g["inputs"], g["param_seed"]
    cfg, params, model = _build(cfg_dict, seed)
    out = model(**_cuda(inp)).cpu()
    ref = fo.flux_forward(params, cfg, **inp, mode="cuda_bf16")
    mask = inp["img_mask"].bool()
    assert rel_l2(out[mask], ref[mask]) < 2e-2
    model.set_lora_mode("merged")
    merged = model(**_cuda(inp)).cpu()
    assert rel_l2(out[mask], merged[mask]) < 1e-2


def test_unmerged_lora_scale_matches_oracle_at_that_scale(ops):
    from oracle import flux_oracle as fo
    g = _load("flux_small_b1.pt")
    cfg, params, model = _build(g["cfg"], g["param_seed"])
    inp = g["inputs"]
    outs = {}
    for s in (0.5, 0.0, 1.0):
        model.set_lora_scale(s)
        outs[s] = model(**_cuda(inp)).cpu()
        ref = fo.flux_forward(params, dataclasses.replace(cfg, lora_scale=s), **inp, mode="cuda_bf16")
        assert rel_l2(outs[s], ref) < 2e-2, s
    assert rel_l2(outs[0.5], outs[0.0]) > 1e-3, "the LoRA branch must contribute"


def _packed_pointers(eng):
    """(struct field path -> (w, lora_a, lora_b) pointers) of every Linear the engine packed."""
    P = eng.params
    out = {}
    top = {"img_in": "img_in", "txt_in": "txt_in", "time_in0": "time_in.in_layer", "time_in1": "time_in.out_layer",
           "vector_in0": "vector_in.in_layer", "vector_in1": "vector_in.out_layer", "final_mod": "final_layer.adaLN_modulation.1",
           "final_linear": "final_layer.linear"}
    if P.guidance_embed:
        top.update(guidance_in0="guidance_in.in_layer", guidance_in1="guidance_in.out_layer")
    for f, n in top.items():
        out[n] = getattr(eng._w, f)
    for i in range(P.depth):
        for s in ("img", "txt"):
            sw = getattr(eng._dbl[i], s)
            for f, n in (("mod", "_mod.lin"), ("qkv", "_attn.qkv"), ("proj", "_attn.proj"), ("mlp0", "_mlp.0"), ("mlp2", "_mlp.2")):
                out[f"double_blocks.{i}.{s}{n}"] = getattr(sw, f)
    for i in range(P.depth_single_blocks):
        for f, n in (("mod", "modulation.lin"), ("linear1", "linear1"), ("linear2", "linear2")):
            out[f"single_blocks.{i}.{n}"] = getattr(eng._sgl[i], f)
    return out


def test_unmerged_engine_is_copy_free(ops):
    cfg_dict, _ = _full_width_case()
    cfg, params, model = _build(cfg_dict, 21, mode="unmerged")
    del params
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated()
    eng = model.engine()
    added = torch.cuda.memory_allocated() - before
    pp = dict(model.named_parameters())
    packed = _packed_pointers(eng)
    assert len(packed) == len([n for n in pp if n.endswith(".lora_A.weight")])
    for name, lw in packed.items():
        assert lw.w == pp[name + ".weight"].data_ptr(), name
        assert lw.lora_a == pp[name + ".lora_A.weight"].data_ptr(), name
        assert lw.lora_b == pp[name + ".lora_B.weight"].data_ptr(), name
        assert lw.rank == pp[name + ".lora_A.weight"].shape[0] and lw.lora_scale == 1.0
    print(f"unmerged engine build adds {added / 2**20:.1f} MiB at full width, depth 1+1")
    assert added < 64 * 2**20, added


def test_adapter_switch_by_assign_is_bitwise_a_fresh_model(ops):
    """Two adapters resident; switching with load_state_dict(..., strict=False, assign=True) rebuilds pointers and biases only
    (no allocation beyond the bias vectors and the output) and gives exactly what a model built with that adapter gives."""
    from oracle import flux_oracle as fo
    g = _load("flux_small_b1.pt")
    cfg, params, model = _build(g["cfg"], g["param_seed"])
    lora_keys = [k for k in params if ".lora_" in k]
    adapters = [{k: v.cuda() for k, v in fo.make_params(cfg, seed=s).items() if k in lora_keys} for s in (101, 202)]
    inp = _cuda(g["inputs"])
    model.load_state_dict(adapters[0], strict=False, assign=True)
    out0 = model(**inp)
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    model.load_state_dict(adapters[1], strict=False, assign=True)
    out1 = model(**inp)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    bias_bytes = sum(4 * model.get_parameter(n + ".weight").shape[0] for n in _packed_pointers(model.engine()))
    assert peak <= 2 * bias_bytes + out1.numel() * 2 + 2**20, (peak, bias_bytes)
    assert not torch.equal(out0, out1)
    _, _, fresh = _build(g["cfg"], g["param_seed"])
    fresh.load_state_dict(adapters[1], strict=False)
    assert torch.equal(fresh(**inp), out1)


def test_unmerged_sampler_trajectory(ops):
    import visualcloze_b200.transport as t
    from oracle import flux_oracle as fo
    from oracle import sampler_oracle as so
    gs = _load("sampler.pt")["shift4"]
    gf = _load("flux_small_b1.pt")
    cfg, params, model = _build(gf["cfg"], gf["param_seed"])
    kw = dict(gs["kwargs"])
    fn = t.Sampler(t.create_transport("Linear", "velocity", do_shift=True)).sample_ode(
        sampling_method="euler", atol=1e-6, rtol=1e-3, reverse=False, **kw)
    traj = fn(gs["x"].cuda(), model.forward, dict(_cuda(gs["inputs"]), cond=gs["cond"].cuda())).cpu()

    def model_fn(x, timesteps, **k):
        return fo.flux_forward(params, cfg, img=x, timesteps=timesteps, **k, mode="cuda_bf16")

    ref = so.sample_ode(gs["x"], model_fn, dict(gs["inputs"], cond=gs["cond"]), num_steps=kw["num_steps"],
                        do_shift=kw["do_shift"], time_shifting_factor=kw["time_shifting_factor"], strength=kw.get("strength"))
    assert rel_l2(traj[-1], ref[-1]) < 5e-2
    assert rel_l2(traj[-1], gs["traj"][-1]) < 5e-2
    assert rel_l2(traj[1], ref[1]) < 1e-2


def test_pipeline_process_images_unmerged(ops):
    """VisualClozeModel(..., lora_mode="unmerged") with the stubs of test_pipeline_process_images_end_to_end: the query crop is
    within the forward tolerance of the merged run."""
    import numpy as np
    from PIL import Image
    from visualcloze_b200 import pipeline as P, vae as V
    g = _load("flux_small_b1.pt")
    _, _, model = _build(g["cfg"], g["param_seed"], mode="merged")
    dec = V.AutoEncoderDecoder(V.AutoEncoderParams(ch=64, ch_mult=[1, 2, 2, 2], num_res_blocks=1), device="cuda").init_synthetic(1)
    t5 = lambda prompts: (0.3 * torch.randn(len(prompts), 24, 64, generator=torch.Generator().manual_seed(len(prompts[0])))).to(BF16).cuda()
    clip = lambda prompts: torch.randn(len(prompts), 32, generator=torch.Generator().manual_seed(7)).to(BF16).cuda()

    def encode(x):
        gg = torch.Generator(device="cuda").manual_seed(int(x.shape[-1]))
        return torch.randn(x.shape[0], 16, x.shape[2] // 8, x.shape[3] // 8, generator=gg, device="cuda")

    def run(mode):
        pipe = P.VisualClozeModel(None, resolution=64, model=model, ae_decoder=dec, t5=t5, clip=clip, encode=encode, lora_mode=mode)
        assert model.lora_mode == mode
        pipe.set_grid_size(2, 3)
        imgs = [[Image.new("RGB", (90, 90), (40 * i, 60 * j, 128)) for j in range(3)] for i in range(2)]
        imgs[1][2] = None
        out = pipe.process_images(imgs, ["layout", "task", "content"], seed=5, cfg=30, steps=4, is_upsampling=False)
        assert len(out) == 1 and out[0].size == (64, 64)
        return torch.from_numpy(np.asarray(out[0], dtype=np.float32))

    merged, unmerged = run("merged"), run("unmerged")
    assert rel_l2(unmerged, merged) < 2e-2


# ------------------------------------------------------------------------------------------------
# full size: FLUX.1-Fill geometry, r = 256, against the unmodified reference modules (oracle/_ref) where they are built
# ------------------------------------------------------------------------------------------------
# measured values are printed and kept as JSON in $VCB_REPORT_DIR (default: the system's temporary directory)
REPORT = os.path.join(os.environ.get("VCB_REPORT_DIR") or tempfile.gettempdir(), "lora_unmerged_fullsize.json")


def _record(key, **vals):
    import json
    os.makedirs(os.path.dirname(REPORT), exist_ok=True)
    data = json.load(open(REPORT)) if os.path.exists(REPORT) else {}
    data[key] = {k: float(v) for k, v in vals.items()}
    json.dump(data, open(REPORT, "w"), indent=1, sort_keys=True)
    print(f"[lora_unmerged] {key}: " + ", ".join(f"{k}={float(v):.4g}" for k, v in vals.items()))


@pytest.fixture(scope="module")
def full():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    from oracle import flux_oracle as fo
    from oracle import ref_runner as rr
    import visualcloze_b200.model as M
    P = M.flux_dev_fill_params()
    with torch.device("cuda"):
        ours = M.FluxLoraWrapper(lora_rank=256, params=P)
    ours.init_synthetic(0)
    sd = dict(ours.state_dict())
    ref = rr.build_flux(dataclasses.asdict(P), 256, sd) if rr.available() else None
    cfg = fo.FluxConfig(**dataclasses.asdict(P), lora_rank=256)
    yield dict(ours=ours, ref=ref, sd=sd, cfg=cfg, fo=fo, rr=rr)
    ours._engine = None
    del ours, ref, sd
    torch.cuda.empty_cache()


def test_fullsize_engine_memory_per_mode(full):
    ours = full["ours"]
    added = {}
    for mode in ("merged", "unmerged"):
        ours._engine = None
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        before = torch.cuda.memory_allocated()
        ours.set_lora_mode(mode)
        ours.engine()
        torch.cuda.synchronize()
        added[mode] = torch.cuda.memory_allocated() - before
    _record("engine_build_bytes", merged=added["merged"], unmerged=added["unmerged"])
    assert added["unmerged"] < 256 * 2**20, added
    assert added["merged"] > 20 * 2**30, added


def test_fullsize_cfgB_forward_unmerged_vs_reference(full):
    import bench
    full["ours"].set_lora_mode("unmerged")
    x, kw, Li, Lt = bench.make_inputs("B", 1234)
    cond = kw.pop("cond")
    inp = _cuda(dict(kw, img=torch.cat((x, cond), dim=-1), timesteps=torch.tensor([0.63])))
    out = full["ours"](**inp).float()
    assert out.shape == (1, Li, 64) and torch.isfinite(out).all()
    fo = full["fo"]
    orc = fo.flux_forward(full["sd"], full["cfg"], **inp, mode="cuda_bf16").float()
    res = dict(ours_unmerged_vs_oracle=rel_l2(out, orc))
    if full["ref"] is not None:
        from test_fullsize_gpu import _MergedView
        ref = full["rr"].flux_forward(full["ref"], **inp).float()
        orc_m = fo.flux_forward(_MergedView(full["sd"]), full["cfg"], **inp, mode="cuda_bf16").float()
        res.update(ours_unmerged_vs_reference=rel_l2(out, ref), floor_unmerged_oracle_vs_reference=rel_l2(orc, ref),
                   floor_merged_oracle_vs_reference=rel_l2(orc_m, ref))
    _record("cfgB_forward_unmerged_19+38_L3968", **res)
    # full depth (57 bf16 blocks): the reference bar below also bounds the distance to the restated oracle
    assert res["ours_unmerged_vs_oracle"] < 2.5e-2, res
    if full["ref"] is None:
        pytest.skip("oracle/_ref absent: compared with the restated oracle only")
    assert res["ours_unmerged_vs_reference"] < 2.5e-2, res
    assert res["ours_unmerged_vs_reference"] < 1.2 * res["floor_merged_oracle_vs_reference"], res


def test_fullsize_cfgB_trajectory_3_evaluations_unmerged(full):
    import bench
    import visualcloze_b200.transport as T
    from oracle import sampler_oracle as so
    full["ours"].set_lora_mode("unmerged")
    x, kw, Li, Lt = bench.make_inputs("B", 1234)
    xg, kwg = x.cuda(), _cuda(kw)
    fn = T.Sampler(T.create_transport("Linear", "velocity", do_shift=True)).sample_ode(
        sampling_method="euler", num_steps=4, atol=1e-6, rtol=1e-3, reverse=False, do_shift=True, time_shifting_factor=1)
    traj = fn(xg, full["ours"].forward, kwg).float()
    assert traj.shape == (4, 1, Li, 64) and torch.equal(traj[0], xg.float())

    def model_fn(inp, timesteps, **k):
        return full["fo"].flux_forward(full["sd"], full["cfg"], img=inp, timesteps=timesteps.cuda(), **k, mode="cuda_bf16")

    orc = so.sample_ode(xg, model_fn, kwg, num_steps=4, do_shift=True, time_shifting_factor=1).float()
    res = dict(final_vs_oracle=rel_l2(traj[-1], orc[-1]), step1_vs_oracle=rel_l2(traj[1], orc[1]))
    if full["ref"] is not None:
        ref = full["rr"].sample_ode(full["ref"], xg, kwg, num_steps=4, do_shift=True, time_shifting_factor=1).float()
        res.update(final_vs_reference=rel_l2(traj[-1], ref[-1]), step1_vs_reference=rel_l2(traj[1], ref[1]))
    _record("cfgB_trajectory_3eval_unmerged", **res)
    assert res["final_vs_oracle"] < 5e-2, res
    if "final_vs_reference" in res:
        assert res["final_vs_reference"] < 5e-2, res
