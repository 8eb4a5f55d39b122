"""Opt-in FP8 (e4m3) projections -- kernel correctness and the parity study that defines their tolerance contract.

The fp8 path is NOT the reference's numerics (the reference computes every Linear in bf16); it exists because the step is
tensor-bound at ~0.8 of the bf16 peak and e4m3 operands double that peak for the 58 % of GEMM FLOPs whose A operand comes out of
an AdaLN LayerNorm (SURVEY.md 8f-3).  Two kinds of checks:

  * kernels: the fp8 GEMM (wgmma e4m3, per-row x per-channel rescale, every epilogue it supports) against an fp32
    matmul of the DEQUANTISED operands -- this isolates the kernel from the quantisation error, tolerance = the bf16 kernels';
    the fp8 LayerNorm against quantising the bf16 LayerNorm kernel's output in torch (scales exact, bytes within 1 e4m3 ulp);
    the row quantiser of level 2 ("fp8_all": attn.proj / mlp.2 / linear2 too) bit for bit against the same rule in torch;
  * contract: block / full-depth forward / multi-step trajectory / decoded image, fp8 (both levels) vs the bf16 path of this
    library on the same weights, written to gpurun_out/fp8_parity.json.  Stated tolerance: forward rel-L2 <= 1.5e-1, trajectory <= 1.5e-1,
    decoded query row PSNR >= 20 dB (random-init weights are a worst case: no trained-weight structure to average over).
"""
import json
import math
import os

import pytest
import torch

from conftest import REPO, rel_l2

pytestmark = pytest.mark.gpu
BF16 = torch.bfloat16
F8 = torch.float8_e4m3fn
REPORT = os.path.join(REPO, "gpurun_out", "fp8_parity.json")


def _record(key, **vals):
    os.makedirs(os.path.dirname(REPORT), exist_ok=True)
    data = json.load(open(REPORT)) if os.path.exists(REPORT) else {}
    data[key] = {k: float(v) for k, v in vals.items()}
    json.dump(data, open(REPORT, "w"), indent=1, sort_keys=True)
    print(f"[fp8] {key}: " + ", ".join(f"{k}={float(v):.3e}" for k, v in vals.items()))


@pytest.fixture(scope="module")
def ops():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    from visualcloze_b200 import ops as o
    return o


def _quant_rows(x):
    s = x.abs().amax(dim=1).clamp_min(1e-12) / 448.0
    return (x / s[:, None]).to(F8), s


@pytest.mark.parametrize("shape", [(256, 256, 512), (3968, 9216, 3072), (520, 384, 1000 + 24), (29, 512, 3072)])
@pytest.mark.parametrize("cfg", [(128, 1), (256, 1), (128, 2), (256, 2)])
def test_gemm_fp8_bias_vs_dequantised_fp32(ops, shape, cfg):
    M, N, K = shape
    bn, cg = cfg
    g = torch.Generator().manual_seed(M + N)
    a32 = torch.randn(M, K, generator=g)
    w32 = torch.randn(N, K, generator=g) / math.sqrt(K)
    a8, sa = _quant_rows(a32)
    w8, sw = _quant_rows(w32)
    bias = torch.randn(N, generator=g)
    out = torch.empty(M, N, dtype=BF16, device="cuda")
    ops.gemm(a8.cuda(), w8.cuda(), bias.cuda(), out, a_scale=sa.cuda(), w_scale=sw.cuda(), block_n=bn, cta_group=cg)
    torch.cuda.synchronize()
    ref = ((a8.float() * sa[:, None]) @ (w8.float() * sw[:, None]).T + bias).to(BF16)
    e = rel_l2(out.cpu(), ref)
    assert e < 4e-3, f"rel_l2 {e:.3e}"


def test_gemm_fp8_gelu_and_grouped(ops):
    """BIAS_GELU epilogue, two problems in one launch, row-mapped output (the mlp.0 launch of a double block)."""
    g = torch.Generator().manual_seed(3)
    K, N, Li, Lt = 512, 1024, 400, 96
    L = Li + Lt
    a32 = torch.randn(L, K, generator=g)
    a8, sa = _quant_rows(a32)
    outs = torch.zeros(L, N + 64, dtype=BF16, device="cuda")
    probs, refs = [], []
    for off, rows in ((Lt, Li), (0, Lt)):
        w8, sw = _quant_rows(torch.randn(N, K, generator=g) / math.sqrt(K))
        bias = torch.randn(N, generator=g)
        probs.append(dict(a=a8.cuda()[off:off + rows], w=w8.cuda(), bias=bias.cuda(), out=outs, epilogue=ops.EPI_BIAS_GELU, out_col_offset=64,
                          rows_per_batch=rows, out_batch_rows=L, out_row_offset=off, a_scale=sa.cuda(), w_scale=sw.cuda()))
        lin = ((a8[off:off + rows].float() * sa[off:off + rows, None]) @ (w8.float() * sw[:, None]).T + bias).to(BF16)
        refs.append((off, rows, torch.nn.functional.gelu(lin.float(), approximate="tanh").to(BF16)))
    ops.gemm_grouped(probs[0], probs[1])
    torch.cuda.synchronize()
    for off, rows, ref in refs:
        assert rel_l2(outs[off:off + rows, 64:].cpu(), ref) < 5e-3
    assert float(outs[:, :64].abs().max()) == 0


def test_gemm_fp8_rejects_unsupported(ops):
    a8 = torch.zeros(128, 256, dtype=F8, device="cuda")
    w8 = torch.zeros(128, 256, dtype=F8, device="cuda")
    out = torch.zeros(128, 128, dtype=BF16, device="cuda")
    with pytest.raises(Exception, match="fp8"):
        ops.gemm(a8, w8, None, out, epilogue=5)                  # VCB_EPI_BIAS_F32 (fp32 scores of the VAE attention): bf16 operands only
    with pytest.raises(Exception, match="fp8"):
        ops.gemm(a8, w8, None, out, block_n=192)


@pytest.mark.parametrize("K", [3072, 12288, 15360, 256, 1032])
def test_quantize_rows_e4m3_bit_exact(ops, K):
    """vcb_quantize_rows_e4m3 on a column window of a wider buffer (the engine quantises cat[:, :H], cat[:, H:] or whole rows):
    scales exactly max|x| / 448, bytes exactly cvt.rn.satfinite.e4m3(x * (1 / s)), nothing outside the window touched."""
    g = torch.Generator().manual_seed(K)
    rows, pad = 333, 64
    buf = (torch.randn(rows, K + 2 * pad, generator=g) * torch.rand(rows, 1, generator=g) * 9).to(BF16).cuda()
    buf[7] = 0                                               # an all-zero row: scale floor 1e-12 / 448, bytes 0
    buf[11, pad + 5] = 3.0e4                                 # an outlier defines its row's scale
    out8 = torch.full((rows, K + 2 * pad), 0.5, dtype=BF16, device="cuda").to(F8)
    rs = torch.full((rows,), -1.0, dtype=torch.float32, device="cuda")
    ops.quantize_rows_e4m3(buf[:, pad:pad + K], out8[:, pad:pad + K], rs)
    torch.cuda.synchronize()
    x = buf[:, pad:pad + K].float()
    s = (x.abs().amax(dim=1).clamp_min(1e-12) * torch.tensor(1.0 / 448.0, device="cuda")).float()
    assert torch.equal(rs, s)
    inv = (1.0 / s).float()
    ref8 = (x * inv[:, None]).clamp(-448, 448).to(F8)
    assert torch.equal(out8[:, pad:pad + K].view(torch.uint8), ref8.view(torch.uint8))
    half = torch.tensor(0.5, dtype=BF16).to(F8).view(torch.uint8).item()
    assert bool((out8[:, :pad].view(torch.uint8) == half).all()) and bool((out8[:, pad + K:].view(torch.uint8) == half).all())
    with pytest.raises(Exception, match="quantize_rows_e4m3"):
        ops.quantize_rows_e4m3(buf[:, :20], out8[:, :20], rs)


@pytest.mark.parametrize("cfg", [(128, 1), (256, 2)])
def test_gemm_fp8_gate_res_with_row_stats(ops, cfg):
    """level 2: the gated-residual epilogue (x += gate * (A W^T + b)) on e4m3 operands, two streams in one launch, residual rows
    mapped into the joint buffer, LayerNorm statistics of the new rows left behind -- vs fp32 math on the dequantised operands."""
    bn, cg = cfg
    g = torch.Generator().manual_seed(9)
    K, N, Li, Lt = 1024, 512, 400, 96
    L = Li + Lt
    a8, sa = _quant_rows(torch.randn(L, K, generator=g))
    x0 = torch.randn(L, N, generator=g).to(BF16)
    x = x0.clone().cuda()
    stats = torch.zeros(L, N // 64, 2, dtype=torch.float32, device="cuda")
    probs, refs = [], []
    for off, rows in ((Lt, Li), (0, Lt)):
        w8, sw = _quant_rows(torch.randn(N, K, generator=g) / math.sqrt(K))
        bias = torch.randn(N, generator=g)
        gate = torch.randn(1, N, generator=g).to(BF16)
        probs.append(dict(a=a8.cuda()[off:off + rows], w=w8.cuda(), bias=bias.cuda(), out=x, epilogue=ops.EPI_GATE_RES, gate=gate.cuda(), res=x,
                          rows_per_batch=rows, out_batch_rows=L, out_row_offset=off, a_scale=sa.cuda(), w_scale=sw.cuda(), row_stats=stats,
                          block_n=bn, cta_group=cg))
        lin = (a8[off:off + rows].float() * sa[off:off + rows, None]) @ (w8.float() * sw[:, None]).T + bias
        refs.append((off, rows, (x0[off:off + rows].float() + gate.float() * lin).to(BF16)))
    ops.gemm_grouped(probs[0], probs[1])
    torch.cuda.synchronize()
    for off, rows, ref in refs:
        assert rel_l2(x[off:off + rows].cpu(), ref) < 5e-3
    xf = x.float().reshape(L, N // 64, 64)
    assert torch.allclose(stats[..., 0], xf.sum(-1), rtol=1e-3, atol=2e-2) and torch.allclose(stats[..., 1], (xf * xf).sum(-1), rtol=2e-3, atol=2e-2)


def test_ln_modulate_fp8_matches_quantised_bf16_kernel(ops):
    g = torch.Generator().manual_seed(5)
    rows, H = 1000, 3072
    x = (torch.randn(rows, H, generator=g) * 1.7 + 0.3).to(BF16).cuda()
    shift = (0.2 * torch.randn(1, H, generator=g)).to(BF16).cuda()
    scale = (0.3 * torch.randn(1, H, generator=g)).to(BF16).cuda()
    y = torch.empty(rows, H, dtype=BF16, device="cuda")
    ops.ln_modulate(x, shift, scale, y, rows_per_batch=rows)
    y8 = torch.empty(rows, H, dtype=F8, device="cuda")
    rs = torch.zeros(rows, dtype=torch.float32, device="cuda")
    ops.ln_modulate_fp8(x, shift, scale, y8, rs, rows_per_batch=rows)
    torch.cuda.synchronize()
    s_ref = y.float().abs().amax(dim=1) / 448.0
    assert torch.allclose(rs, s_ref, rtol=1e-6, atol=0), "row scale must be max|bf16(y)| / 448"
    deq = y8.float() * rs[:, None]
    # e4m3 has 3 mantissa bits: relative step 2^-3 at the top of a binade, i.e. rounding error <= 2^-4 of the value (+ denormal floor)
    err = (deq - y.float()).abs()
    assert bool((err <= y.float().abs() * 2.0 ** -4 + rs[:, None] * 2.0 ** -9 * 1.01).all())
    assert rel_l2(deq, y.float()) < 4e-2
    # statistics supplied by the producer (what the GATE_RES epilogue leaves behind): same bytes up to the statistics' fp32 rounding
    xf = x.float().reshape(rows, H // 64, 64)
    stats = torch.stack((xf.sum(-1), (xf * xf).sum(-1)), dim=-1).contiguous()
    y8s = torch.empty(rows, H, dtype=F8, device="cuda")
    rs2 = torch.zeros(rows, dtype=torch.float32, device="cuda")
    ops.ln_modulate_fp8(x, shift, scale, y8s, rs2, rows_per_batch=rows, stats=stats)
    torch.cuda.synchronize()
    assert torch.allclose(rs2, rs, rtol=2e-2, atol=0)        # a row maximum may land on the neighbouring bf16 value
    assert rel_l2(y8s.float() * rs2[:, None], deq) < 2e-2


@pytest.fixture(scope="module")
def pair():
    """the same full-width weights packed twice: bf16 projections and fp8 projections"""
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    import dataclasses
    import visualcloze_b200.model as M
    P = dataclasses.replace(M.flux_dev_fill_params(), depth=2, depth_single_blocks=4)
    with torch.device("cuda"):
        m = M.FluxLoraWrapper(lora_rank=64, params=P)
    m.init_synthetic(3)
    return m


def _inputs(workload="A"):
    import bench
    x, kw, Li, Lt = bench.make_inputs(workload, 1234)
    return x, kw, Li


def test_fp8_forward_reduced_depth_vs_bf16(pair):
    """2 + 4 blocks at full width (hidden 3072, 24 heads), cfg-A tokens: fp8 vs bf16 projections on the same weights"""
    x, kw, Li = _inputs("A")
    cond = kw.pop("cond")
    inp = {k: (v.cuda() if torch.is_tensor(v) else v) for k, v in dict(kw, img=torch.cat((x, cond), -1), timesteps=torch.tensor([0.6])).items()}
    pair.set_linear_precision("bf16")
    ref = pair(**inp).float()
    pair.set_linear_precision("fp8")
    out = pair(**inp).float()
    pair.set_linear_precision("fp8_all")
    out2 = pair(**inp).float()
    pair.set_linear_precision("bf16")
    again = pair(**inp).float()
    assert torch.equal(again, ref), "switching back must restore the bf16 path bit for bit"
    e, e2 = rel_l2(out, ref), rel_l2(out2, ref)
    _record("forward_2+4_blocks_cfgA", rel_l2_fp8_vs_bf16=e, rel_l2_fp8_all_vs_bf16=e2)
    assert torch.isfinite(out).all() and 1e-4 < e < 1e-1, e
    assert torch.isfinite(out2).all() and e < e2 < 1.5e-1, (e, e2)          # more Linears quantised: further from bf16, same order


@pytest.mark.parametrize("precision", ["fp8", "fp8_all"])
def test_fp8_ragged_batch_matches_bf16_on_valid_tokens(precision):
    """batch 2 with different image lengths (the reference golden's ragged case, tests/golden/flux_small_b2r.pt): padded rows are
    don't-care, valid rows of the fp8 paths stay finite and close to the bf16 path -- the row quantiser and the per-row scales
    must follow the physical row mapping of the joint buffer for every sample."""
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    import visualcloze_b200.model as M
    from test_flux_gpu import _build, _load
    g = _load("flux_small_b2r.pt")
    cfg, params, model = _build(M, g["cfg"], g["param_seed"])
    inp = {k: (v.cuda() if torch.is_tensor(v) else v) for k, v in g["inputs"].items()}
    ref = model(**inp).float()
    model.set_linear_precision(precision)
    out = model(**inp).float()
    mask = inp["img_mask"].bool()
    assert bool(torch.isfinite(out[mask]).all())
    e = rel_l2(out[mask], ref[mask])
    for b in range(mask.shape[0]):                       # per sample: a wrong row mapping would wreck one sample, not the average
        eb = rel_l2(out[b][mask[b]], ref[b][mask[b]])
        assert 0 < eb < 1.5e-1, (precision, b, eb)
    _record(f"ragged_b2_small_{precision}", rel_l2_vs_bf16=e)


def test_fp8_full_depth_forward_trajectory_and_image():
    """cfg B, full depth 19 + 38: one evaluation, a 5-evaluation trajectory and the decoded query row, fp8 vs bf16 projections"""
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    import visualcloze_b200.model as M
    import visualcloze_b200.transport as T
    from visualcloze_b200 import vae as V
    with torch.device("cuda"):
        m = M.FluxLoraWrapper(lora_rank=256, params=M.flux_dev_fill_params())
    m.init_synthetic(0)
    dec = V.AutoEncoderDecoder(device="cuda").init_synthetic(0)
    x, kw, Li = _inputs("B")
    xg, kwg = x.cuda(), {k: v.cuda() for k, v in kw.items()}
    fn = T.Sampler(T.create_transport("Linear", "velocity", do_shift=True)).sample_ode(
        sampling_method="euler", num_steps=6, atol=1e-6, rtol=1e-3, reverse=False, do_shift=True, time_shifting_factor=1)
    res = {}
    outs = {}
    for prec in ("bf16", "fp8", "fp8_all"):
        m.set_linear_precision(prec)
        one = m(**dict({k: v for k, v in kwg.items() if k != "cond"}, img=torch.cat((xg, kwg["cond"]), -1), timesteps=torch.tensor([0.63]).cuda())).float()
        traj = fn(xg, m.forward, kwg).float()
        row = Li // 2
        img = dec.decode_packed(traj[-1][:, Li - row:, :].to(BF16), 384 // 16, 3 * 384 // 16).float()
        outs[prec] = (one, traj, img)
    for prec in ("fp8", "fp8_all"):
        res = dict(forward_rel_l2=rel_l2(outs[prec][0], outs["bf16"][0]),
                   trajectory_final_rel_l2=rel_l2(outs[prec][1][-1], outs["bf16"][1][-1]))
        mse = (outs[prec][2] - outs["bf16"][2]).pow(2).mean().item()
        res["query_row_psnr_db"] = 10 * math.log10(255.0 ** 2 / max(mse, 1e-12))
        _record(f"cfgB_full_depth_{prec}_vs_bf16", **res)
        assert res["forward_rel_l2"] < 1.5e-1 and res["trajectory_final_rel_l2"] < 1.5e-1 and res["query_row_psnr_db"] >= 20.0, (prec, res)
