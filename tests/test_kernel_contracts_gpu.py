"""The GEMM, implicit-GEMM convolution and joint-attention kernels element by element against the references of
tests/kernel_contract_ref.py: bit for bit where the operands make the result exactly known, inside stated intervals / bounds
elsewhere, and with canary-filled margins around every output (rows above and below, columns on both sides, ldo wider than the
problem) that must come back untouched."""
import math
import os
import subprocess
import sys

import pytest
import torch

import kernel_contract_ref as kr

pytestmark = pytest.mark.gpu

BF16, F32 = torch.bfloat16, torch.float32
GRAIN = 2.0 ** -5                      # a in {-7..7} 2^-2, w in {-7..7} 2^-3: every product is a multiple of 2^-5
TOP, BOTTOM, LEFT, RIGHT = 3, 2, 16, 24


@pytest.fixture(scope="module")
def ops():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    from visualcloze_b200 import ops as _ops
    return _ops


def _ru(x, m):
    return (x + m - 1) // m * m


# ----------------------------------------------------------------------------------------------
# GEMM, bf16 operands: a pairwise-covering case list
# ----------------------------------------------------------------------------------------------
CONFIGS = [(64, 1), (128, 1), (192, 1), (256, 1), (128, 2), (192, 2), (256, 2)]
MS = [1, 63, 64, 65, 129, 255, 257]
KS = [8, 72, 1000, 3072]
PLAIN_EPIS = ["bias", "gelu", "gate", "res", "f32"]
HEAD_EPIS = PLAIN_EPIS + ["qkv", "linear1"]


def _n_for(epi, bn, j):
    if epi == "bias":
        return [13, 261, bn - 8, bn + 8, 520][j % 5]
    if epi == "f32":                                     # N % 8 in 1..4: fp32 stores stop at round_up(N, 4) < round_up(N, 8)
        return [12, 258, bn + 4, 261, 260][j % 5]
    if epi in ("gelu", "gate", "res"):
        return [bn - 8, bn + 8, 520][j % 3]
    if epi == "qkv":
        return [384, 768][j % 2]
    return [384 + 128, 768 + 256][j % 2]                 # linear1: 3H + mlp


def gemm_cases():
    """every (block_n, cta_group) meets every M level, every K level and every epilogue its tile allows; N, batching, alpha,
    LoRA rank and the residual layout rotate with different strides"""
    cases = []
    for ci, (bn, cg) in enumerate(CONFIGS):
        epis = HEAD_EPIS if bn % 128 == 0 else PLAIN_EPIS
        for i, M in enumerate(MS):
            epi = epis[(i + ci) % len(epis)]
            cases.append(dict(
                epi=epi, bn=bn, cg=cg, rows=M, N=_n_for(epi, bn, i + 2 * ci), K=KS[(i + 2 * ci) % 4],
                batch=3 if (i + ci) % 2 else 1, row_off=[0, 5, 1][(i + ci) % 3], a_pad=[0, 3][(i + 2 * ci) % 2],
                alpha=[0.0, 0.5, 0.7][(i + 3 * ci) % 3], rank=[0, 0, 8, 64, 72][(i + ci) % 5], res_sep=(i + ci) % 3 == 2,
                seed=100 * ci + i))
    return cases


CASES = gemm_cases()


def _case_id(c):
    return f"{c['epi']}-bn{c['bn']}cg{c['cg']}-M{c['rows']}x{c['batch']}-N{c['N']}-K{c['K']}-r{c['rank']}-a{c['alpha']}"


def run_gemm_case(ops, epi, bn, cg, rows, N, K, batch=1, row_off=0, a_pad=0, alpha=0.0, rank=0, res_sep=False, seed=0,
                  slack=2, stats=False):
    """One launch with exact operands, canary-margined outputs and garbage where the kernel must not read (A / W columns past K,
    A rows between samples); returns a list of failure descriptions (empty = the kernel kept the contract)."""
    g = torch.Generator().manual_seed(seed)
    lda = _ru(K, 8) + 8
    rs = rows + a_pad                                     # rows per sample in A's storage (a_batch_stride > rows * lda)
    A = kr.exact_bf16((batch * rs, lda), g, 2)
    W = kr.exact_bf16((N, lda), g, 3)
    A[:, K:] = 1e4                                        # must never reach the accumulator (TMA zero-fills the k tail)
    W[:, K:] = -1e4
    if a_pad:
        for b in range(batch):
            A[b * rs + rows:(b + 1) * rs] = 3e4
    a_rows = torch.cat([A[b * rs:b * rs + rows, :K] for b in range(batch)])
    acc = kr.exact_acc(a_rows, W[:, :K], GRAIN)
    lora = {}
    if rank:
        T = kr.exact_bf16((batch * rs, rank), g, 2)
        Lb = kr.exact_bf16((N, rank), g, 3)
        t_rows = torch.cat([T[b * rs:b * rs + rows] for b in range(batch)])
        acc = kr.exact_acc(torch.cat([a_rows, t_rows], 1), torch.cat([W[:, :K], Lb], 1), GRAIN)
        lora = dict(lora_t=T.cuda(), lora_b=Lb.cuda(), lora_t_batch_stride=rs * rank if batch > 1 else 0)
    acc = kr.scale_acc(acc, alpha)
    bias = torch.randn(N, generator=g)
    obr = row_off + rows + slack                          # out_batch_rows > rows_per_batch
    out_rows = batch * obr
    f32 = epi == "f32"
    dt = F32 if f32 else BF16
    ncols = N if epi != "linear1" else 3 * (N // 4)       # linear1: out holds the 3H q/k/v columns, out2 the mlp
    ldo = LEFT + _ru(ncols, 8) + RIGHT
    buf = kr.canary_like(TOP + out_rows + BOTTOM, ldo, dt)
    orow = torch.cat([torch.arange(rows) + b * obr + row_off for b in range(batch)])      # mapped output row of every A row
    kw = dict(epilogue={"bias": ops.EPI_BIAS, "gelu": ops.EPI_BIAS_GELU, "gate": ops.EPI_GATE_RES, "res": ops.EPI_GATE_RES,
                        "f32": ops.EPI_BIAS_F32, "qkv": ops.EPI_QKV, "linear1": ops.EPI_LINEAR1}[epi],
              out_col_offset=LEFT, rows_per_batch=rows, out_batch_rows=obr, out_row_offset=row_off, block_n=bn, cta_group=cg,
              a_batch_stride=rs * lda if batch > 1 else 0, m=batch * rows, alpha=alpha, **lora)
    want = buf.clone()
    region = torch.zeros(want.shape, dtype=torch.bool)
    lo = hi = None
    extra = []
    gate_rows = res_rows = None
    if epi in ("gate", "res"):
        res_vals = torch.randn(out_rows, ldo, generator=g).to(BF16)
        if res_sep:
            ld_res = ldo + 40                             # its own leading dimension
            res_buf = torch.randn(out_rows + 4, ld_res, generator=g).to(BF16)
            res_gpu = res_buf.cuda()
            kw["res"] = res_gpu[:out_rows, LEFT:]         # indexed by output row, columns from 0
            res_rows = res_buf[orow, LEFT:LEFT + N]
            extra.append(("res", res_gpu, res_buf))
        else:
            # res aliases out: res values in the problem region only, canaries everywhere beside it
            buf[TOP + orow, LEFT:LEFT + N] = res_vals[orow, LEFT:LEFT + N]
            want = buf.clone()
            res_rows = res_vals[orow, LEFT:LEFT + N]
        if epi == "gate":
            mod = torch.randn(batch, 6 * N, generator=g).to(BF16)       # the engine's [B, 6H] modulation rows
            gate_gpu = mod.cuda()[:, 2 * N:3 * N]
            kw["gate"] = gate_gpu
            gate_rows = mod[:, 2 * N:3 * N].repeat_interleave(rows, 0)
    out = buf.cuda()
    outv = out[TOP:TOP + out_rows]
    if "res" in (epi,) or epi == "gate":
        if not res_sep:
            kw["res"] = outv[:, LEFT:]
            kw["out_col_offset"] = 0
            outv = outv[:, LEFT:]
    if stats:
        sbuf = kr.canary_like(1, (TOP + out_rows + BOTTOM) * (N // 64) * 2, F32)
        sg = sbuf.cuda()
        kw["row_stats"] = sg[0, TOP * (N // 64) * 2:].view(-1, N // 64, 2)[:out_rows]
    R = TOP + orow
    cols = slice(LEFT, LEFT + N)
    if epi == "bias":
        want[R, cols] = kr.epi_bias(acc, bias)
        want[TOP + orow[:, None], torch.arange(LEFT + N, LEFT + _ru(N, 8))[None]] = 0.0
    elif epi == "f32":
        want[R, cols] = kr.epi_bias_f32(acc, bias)
        want[TOP + orow[:, None], torch.arange(LEFT + N, LEFT + _ru(N, 4))[None]] = 0.0      # round_up(N, 4), vcb200.h
    elif epi in ("gate", "res"):
        want[R, cols] = kr.epi_gate_res(acc, bias, gate_rows, res_rows)
    elif epi == "gelu":
        lo, hi = want.clone(), want.clone()
        lo[R, cols], hi[R, cols] = kr.epi_gelu_interval(acc, bias)
        region[R, cols] = True
    else:
        H = N // 3 if epi == "qkv" else N // 4
        rope_rows = out_rows
        ang = torch.randn(rope_rows, 64, generator=g) * 3
        cos, sin = torch.cos(ang), torch.sin(ang)
        rope = torch.stack([cos, sin], -1).permute(1, 0, 2).contiguous()
        qs = (1 + 0.25 * torch.randn(128, generator=g)).to(BF16)
        ks = (1 + 0.25 * torch.randn(128, generator=g)).to(BF16)
        kw.update(hidden=H, q_scale=qs.cuda(), k_scale=ks.cuda(), rope=rope.cuda())
        lin = kr.linear_bf16(acc, bias)
        lo, hi = want.clone(), want.clone()
        qlo, qhi = kr.qkv_interval(lin[:, :3 * H], qs, ks, cos[orow], sin[orow], H)
        c3 = slice(LEFT, LEFT + 3 * H)
        lo[R, c3], hi[R, c3] = qlo, qhi
        region[R, c3] = True
        if epi == "linear1":
            mlp = N - 3 * H
            ld2 = 8 + mlp + 16
            buf2 = kr.canary_like(TOP + out_rows + BOTTOM, ld2, BF16)
            out2 = buf2.cuda()
            kw.update(out2=out2[TOP:TOP + out_rows], out2_col_offset=8)
            lo2, hi2 = buf2.clone(), buf2.clone()
            glo, ghi = kr.epi_gelu_interval(acc[:, 3 * H:], bias[3 * H:])
            lo2[R, 8:8 + mlp], hi2[R, 8:8 + mlp] = glo, ghi
            reg2 = torch.zeros(buf2.shape, dtype=torch.bool)
            reg2[R, 8:8 + mlp] = True
            extra.append(("out2", out2, (lo2, hi2, reg2)))
    w_gpu = W.cuda()
    ops.gemm(A.cuda()[:, :K], w_gpu[:, :K], bias.cuda(), outv, **kw)
    torch.cuda.synchronize()
    errs = []
    got = out.cpu()
    what = f"{epi} bn={bn} cg={cg} rows={rows} batch={batch} N={N} K={K} rank={rank} alpha={alpha}"
    e = kr.check_exact(got, want, what) if lo is None else kr.check_interval(got, lo, hi, region, what)
    if e:
        errs.append(e)
    for name, t, ref in extra:
        if name == "res":
            e = kr.check_exact(t.cpu(), ref, what + " (separate res must come back unchanged)")
        else:
            e = kr.check_interval(t.cpu(), *ref, what + " (out2)")
        if e:
            errs.append(e)
    if stats:
        sgot = sg.cpu()
        per = (N // 64) * 2
        st = sgot[0, TOP * per:(TOP + out_rows) * per].view(out_rows, N // 64, 2).to(torch.float64)
        x = got[TOP:TOP + out_rows, LEFT:LEFT + N].to(torch.float64).view(out_rows, N // 64, 64)
        rowmask = torch.zeros(out_rows, dtype=torch.bool)
        rowmask[orow] = True
        s1, s2 = x.sum(-1), (x * x).sum(-1)
        tol1, tol2 = 64 * 2.0 ** -24 * x.abs().sum(-1), 64 * 2.0 ** -24 * s2
        ok = ((st[..., 0] - s1).abs() <= tol1) & ((st[..., 1] - s2).abs() <= tol2)
        if not bool(ok[rowmask].all()):
            errs.append(f"{what}: row_stats outside 64 * 2^-24 * sum|x| for {int((~ok[rowmask]).sum())} slots")
        sb = kr.bits(sgot).view(TOP + out_rows + BOTTOM, per)
        keep = torch.ones(TOP + out_rows + BOTTOM, dtype=torch.bool)
        keep[TOP + orow] = False
        if not bool(sb[keep].eq(kr.CANARY_F32).all()):
            errs.append(f"{what}: row_stats written outside the problem's rows")
    return errs


@pytest.mark.parametrize("case", CASES, ids=[_case_id(c) for c in CASES])
def test_gemm_contract(ops, case):
    errs = run_gemm_case(ops, **case)
    assert not errs, "\n".join(errs)


@pytest.mark.parametrize("cfg", [(128, 1), (256, 1), (128, 2), (256, 2)])
def test_gemm_row_stats(ops, cfg):
    """row_stats: per output row and 64 columns the (sum, sum of squares) of the stored bf16 values, within 64 2^-24 sum|x|; the
    slots of rows outside the problem keep their canaries"""
    bn, cg = cfg
    errs = run_gemm_case(ops, "gate", bn, cg, rows=129, N=512, K=1000, batch=3, row_off=5, seed=7 + bn + cg, stats=True)
    errs += run_gemm_case(ops, "res", bn, cg, rows=65, N=768, K=72, batch=1, row_off=1, res_sep=True, seed=9 + bn, stats=True)
    assert not errs, "\n".join(errs)


@pytest.mark.parametrize("cfg", [(256, 1), (128, 2)])
@pytest.mark.parametrize("epi", ["bias", "gate"])
def test_gemm_multi_wave(ops, cfg, epi):
    """3000 x 3072: at least twice as many tiles as CTAs (pairs), so every CTA runs two tiles or more"""
    bn, cg = cfg
    M, N = 3000, 3072
    slots = torch.cuda.get_device_properties(0).multi_processor_count // cg
    assert _ru(M, 128 * cg) // (128 * cg) * _ru(N, bn) // bn >= 2 * slots
    errs = run_gemm_case(ops, epi, bn, cg, rows=M, N=N, K=200, seed=31 + bn)
    assert not errs, "\n".join(errs)


@pytest.mark.parametrize("alpha", [0.25, 0.3])
@pytest.mark.parametrize("rank", [8, 64, 72])
def test_gemm_lora_tail_and_alpha(ops, rank, alpha):
    errs = run_gemm_case(ops, "bias", 256, 2, rows=300, N=520, K=1000, batch=1, alpha=alpha, rank=rank, seed=rank)
    errs += run_gemm_case(ops, "gate", 128, 1, rows=65, N=264, K=72, batch=3, alpha=alpha, rank=rank, seed=rank + 1)
    assert not errs, "\n".join(errs)


def test_gemm_grouped_one_row_problem(ops):
    """grouped launch: an img problem of 200 rows and a txt problem of ONE row per sample writing interleaved rows of one joint
    buffer, gated residual in place, gate rows in the [B, 6H] layout"""
    g = torch.Generator().manual_seed(5)
    B, Li, Lt, N, K = 3, 200, 1, 264, 1000
    L = Li + Lt
    ldo = LEFT + N + RIGHT
    A = kr.exact_bf16((B * L, _ru(K, 8) + 8), g, 2)
    buf = kr.canary_like(TOP + B * L + BOTTOM, ldo, BF16)
    buf[TOP:TOP + B * L, LEFT:LEFT + N] = torch.randn(B * L, N, generator=g).to(BF16)      # res in place; canaries beside it
    want = buf.clone()
    out = buf.cuda()
    xv = out[TOP:TOP + B * L, LEFT:]
    Ag = A.cuda()
    probs = []
    for s, (off, rows) in enumerate(((Lt, Li), (0, Lt))):
        W = kr.exact_bf16((N, K), g, 3)
        bias = torch.randn(N, generator=g)
        mod = torch.randn(B, 6 * N, generator=g).to(BF16)
        probs.append(dict(a=Ag[off:, :K], w=W.cuda(), bias=bias.cuda(), out=xv, epilogue=ops.EPI_GATE_RES, m=B * rows, rows_per_batch=rows,
                          out_batch_rows=L, out_row_offset=off, a_batch_stride=L * A.shape[1], gate=mod.cuda()[:, 5 * N:6 * N], res=xv,
                          block_n=128, cta_group=2))
        idx = torch.cat([torch.arange(rows) + b * L + off for b in range(B)])
        acc = kr.exact_acc(A[idx, :K], W, GRAIN)
        want[TOP + idx, LEFT:LEFT + N] = kr.epi_gate_res(acc, bias, mod[:, 5 * N:].repeat_interleave(rows, 0),
                                                          buf[TOP + idx, LEFT:LEFT + N])
    ops.gemm_grouped(probs[0], probs[1])
    torch.cuda.synchronize()
    e = kr.check_exact(out.cpu(), want, "grouped")
    assert e is None, e


SUBSET = [c for c in CASES if c["K"] >= 1000][::2]


def streamk_cases():
    """Every epilogue on every (block_n, cta_group) the stream-K tail serves, at shapes where VCB_STREAMK=1 takes it: one partial
    wave of tiles (3 samples of 257 rows) with at least slots / 7 tiles (capi.cu streamk_feasible) and K = 4096, so that the idle
    part of the wave costs more than 20 us (streamk_wanted).  The child process checks each launch's profile record for the
    stream-K mark rather than trusting this arithmetic."""
    n_plain = {(128, 1): 520, (192, 1): 520, (256, 1): 520, (128, 2): 264, (192, 2): 520, (256, 2): 520}
    n_head = {128: {"qkv": 384, "linear1": 512}, 256: {"qkv": 768, "linear1": 1024}}
    cases = []
    for ci, ((bn, cg), n) in enumerate(n_plain.items()):
        epis = HEAD_EPIS if bn % 128 == 0 else PLAIN_EPIS
        for i, epi in enumerate(epis):
            N = n_head[bn][epi] if epi in ("qkv", "linear1") else (n - 4 if epi == "f32" else n)
            cases.append(dict(epi=epi, bn=bn, cg=cg, rows=257, N=N, K=4096, batch=3, row_off=[0, 5][i % 2], a_pad=[0, 3][(i + ci) % 2],
                              alpha=[0.0, 0.7][(i + ci) % 2], res_sep=(i + ci) % 2 == 1, seed=500 + 10 * ci + i))
    return cases


def test_gemm_contract_streamk_subprocess():
    """The stream-K policy is read once per process: in a child process with VCB_STREAMK=1, every epilogue on every stream-K
    configuration, each launch confirmed to have taken the tail (bit 25 of its profile record).  Stream-K folds exact fp32
    partial sums, so the bit-exact bar holds there too."""
    here = os.path.dirname(os.path.abspath(__file__))
    code = f"""
import sys
sys.path.insert(0, {here!r}); sys.path.insert(0, {os.path.dirname(here)!r})
import test_kernel_contracts_gpu as t
from visualcloze_b200 import ops, _lib
errs = []
for c in t.streamk_cases():
    _lib.lib().vcb_profile_begin()
    errs += t.run_gemm_case(ops, **c)
    _, recs = _lib.profile_end(16)
    gemms = [r for r in recs if r.category == 0]
    if len(gemms) != 1 or not (gemms[0].info[3] >> 25) & 1:
        errs.append(f"stream-K tail not taken for {{c}}: {{[list(r.info) for r in gemms]}}")
print("\\n".join(errs) if errs else "contract ok")
"""
    r = subprocess.run([sys.executable, "-c", code], env=dict(os.environ, VCB_STREAMK="1"), capture_output=True, text=True, timeout=900)
    assert r.returncode == 0 and "contract ok" in r.stdout, r.stdout[-4000:] + r.stderr[-4000:]


def test_gemm_contract_raster_subprocess():
    """The N-fastest raster is read once per process: rerun the long-K half of the case list in a child process with it."""
    here = os.path.dirname(os.path.abspath(__file__))
    code = f"""
import sys
sys.path.insert(0, {here!r}); sys.path.insert(0, {os.path.dirname(here)!r})
import test_kernel_contracts_gpu as t
from visualcloze_b200 import ops
errs = []
for c in t.SUBSET:
    errs += t.run_gemm_case(ops, **c)
print("\\n".join(errs) if errs else "contract ok")
"""
    r = subprocess.run([sys.executable, "-c", code], env=dict(os.environ, VCB_GEMM_RASTER="1"), capture_output=True, text=True, timeout=900)
    assert r.returncode == 0 and "contract ok" in r.stdout, r.stdout[-4000:] + r.stderr[-4000:]


# ----------------------------------------------------------------------------------------------
# GEMM, e4m3 operands
# ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cfg", [(128, 1), (256, 1), (128, 2), (256, 2)])
@pytest.mark.parametrize("epi", ["bias", "gelu", "gate", "qkv", "linear1"])
def test_gemm_fp8_contract(ops, epi, cfg):
    """integer e4m3 operands (|x| <= 4, every partial sum an integer below 2^12 in magnitude at K = 192), power-of-two a_scale /
    w_scale: bit for bit except the GELU / QKV intervals (no intermediate bf16 roundings on this path, tanh.approx GELU);
    non-power-of-two scales: within 1 bf16 ulp of the exact result"""
    bn, cg = cfg
    g = torch.Generator().manual_seed(bn + cg)
    rows, K = 129, 192
    N = {"bias": bn + 16, "gelu": 2 * bn, "gate": bn + 16, "qkv": 384, "linear1": 512}[epi]
    a, w = kr.exact_e4m3((rows, K), g), kr.exact_e4m3((N, K), g)
    acc = kr.exact_acc(a.to(F32), w.to(F32), 1.0)
    assert float((a.to(torch.float64).abs() @ w.to(torch.float64).abs().T).max()) < 2 ** 12
    for pow2 in (True, False):
        if pow2:
            sa = 2.0 ** torch.randint(-3, 2, (rows,), generator=g).float()
            sw = 2.0 ** torch.randint(-4, 1, (N,), generator=g).float()
        else:
            sa = torch.rand(rows, generator=g) + 0.5
            sw = torch.rand(N, generator=g) * 0.1 + 0.01
        bias = torch.randn(N, generator=g)
        scale = sa[:, None] * sw[None, :]
        lin = (acc.double() * scale.double() + bias.double()).float()      # the kernel's fmaf(acc, sa * sw, bias)
        ldo = LEFT + N + RIGHT
        buf = kr.canary_like(TOP + rows + BOTTOM, ldo, BF16)
        kw = dict(block_n=bn, cta_group=cg, a_scale=sa.cuda(), w_scale=sw.cuda())
        H = N // 3 if epi == "qkv" else N // 4
        if epi == "gate":
            buf[TOP:TOP + rows, LEFT:LEFT + N] = torch.randn(rows, N, generator=g).to(BF16)
            gate = torch.randn(1, N, generator=g).to(BF16)
        want = buf.clone()
        out = buf.cuda()
        outv = out[TOP:TOP + rows, LEFT:]
        R, cols = slice(TOP, TOP + rows), slice(LEFT, LEFT + N)
        if epi == "bias":
            ops.gemm(a.cuda(), w.cuda(), bias.cuda(), outv, **kw)
            want[R, cols] = lin.to(BF16)
            cands = [want]
        elif epi == "gate":
            ops.gemm(a.cuda(), w.cuda(), bias.cuda(), outv, epilogue=ops.EPI_GATE_RES, gate=gate.cuda(), res=outv, **kw)
            u, f = kr.epi_gate_res_fp8(acc, scale, bias, gate.expand(rows, N), buf[R, cols])
            cands = []
            for c in (u, f):
                wc = want.clone()
                wc[R, cols] = c
                cands.append(wc)
        else:
            lo, hi = want.clone(), want.clone()
            region = torch.zeros(want.shape, dtype=torch.bool)
            if epi == "gelu":
                lo[R, cols], hi[R, cols] = kr.gelu_interval(lin, fast=True)
                region[R, cols] = True
                ops.gemm(a.cuda(), w.cuda(), bias.cuda(), outv, epilogue=ops.EPI_BIAS_GELU, **kw)
            else:
                ang = torch.randn(rows, 64, generator=g) * 3
                cos, sin = torch.cos(ang), torch.sin(ang)
                rope = torch.stack([cos, sin], -1).permute(1, 0, 2).contiguous()
                qs, ks = (1 + 0.25 * torch.randn(128, generator=g)).to(BF16), (1 + 0.25 * torch.randn(128, generator=g)).to(BF16)
                c3 = slice(LEFT, LEFT + 3 * H)
                lo[R, c3], hi[R, c3] = kr.qkv_interval(lin[:, :3 * H], qs, ks, cos, sin, H, rounded=False)
                region[R, c3] = True
                extra = {}
                if epi == "linear1":
                    buf2 = kr.canary_like(TOP + rows + BOTTOM, 8 + (N - 3 * H) + 16, BF16)
                    out2 = buf2.cuda()
                    extra = dict(out2=out2[TOP:TOP + rows], out2_col_offset=8)
                ops.gemm(a.cuda(), w.cuda(), bias.cuda(), outv, epilogue=ops.EPI_QKV if epi == "qkv" else ops.EPI_LINEAR1, hidden=H,
                         q_scale=qs.cuda(), k_scale=ks.cuda(), rope=rope.cuda(), **extra, **kw)
                if epi == "linear1":
                    lo2, hi2 = buf2.clone(), buf2.clone()
                    reg2 = torch.zeros(buf2.shape, dtype=torch.bool)
                    lo2[R, 8:8 + N - 3 * H], hi2[R, 8:8 + N - 3 * H] = kr.gelu_interval(lin[:, 3 * H:], fast=True)
                    reg2[R, 8:8 + N - 3 * H] = True
                    torch.cuda.synchronize()
                    e = kr.check_interval(out2.cpu(), lo2, hi2, reg2, f"fp8 linear1 out2 {cfg} pow2={pow2}")
                    assert e is None, e
            torch.cuda.synchronize()
            e = kr.check_interval(out.cpu(), lo, hi, region, f"fp8 {epi} {cfg} pow2={pow2}")
            assert e is None, e
            continue
        torch.cuda.synchronize()
        got = out.cpu()
        if pow2:
            errs = [kr.check_exact(got, c, f"fp8 {epi} {cfg}") for c in cands]
            assert any(e is None for e in errs), errs[0]
        else:
            # lin is fp32-exact up to one rounding of acc * scale: the stored bf16 lies within one bf16 ulp of it
            inside = torch.zeros(got.shape, dtype=torch.bool)
            inside[R, cols] = True
            assert bool((kr.bits(got) == kr.bits(want))[~inside].all()), f"fp8 {epi} {cfg}: written outside the output region"
            ref = torch.stack([c[R, cols].double() for c in cands])
            d = (got[R, cols].double()[None] - ref).abs().amin(0)
            ulp = 2.0 ** (torch.floor(torch.log2(ref[0].abs().clamp_min(2.0 ** -126))) - 7)
            assert bool((d <= ulp).all()), f"fp8 {epi} {cfg}: {int((d > ulp).sum())} elements more than 1 bf16 ulp off"


# ----------------------------------------------------------------------------------------------
# implicit-GEMM 3x3 convolution
# ----------------------------------------------------------------------------------------------
def _conv_cases():
    """stride 1 at H, W in {1, 7, 9, 16, 17, 33}; stride 2 at twice those (the entry point takes even inputs only), i.e. odd and
    even OUTPUT sizes 1 .. 33"""
    cases = []
    sizes = [1, 7, 9, 16, 17, 33]
    i = 0
    for stride in (1, 2):
        for j, s in enumerate(sizes):
            H = s * stride
            W = sizes[(j + 2) % len(sizes)] * stride
            cases.append((stride, H, W, [64, 192][i % 2], [8, 24, 264][i % 3], [1, 3][(i // 2) % 2], i % 2 == 1))
            i += 1
    return cases


@pytest.mark.parametrize("case", _conv_cases(), ids=lambda c: "s{}-H{}-W{}-ci{}-co{}-n{}-res{}".format(*c))
def test_conv3x3_contract(ops, case):
    """vcb_conv3x3_nhwc bit for bit against F.conv2d in fp32 on exact operands (+ bias, bf16, + res), canaries before and after
    the NHWC output"""
    from visualcloze_b200 import _lib
    stride, H, W, ci, co, n, with_res = case
    g = torch.Generator().manual_seed(H * 100 + W + ci + co)
    x = kr.exact_bf16((n, ci, H, W), g, 2)
    w = kr.exact_bf16((co, ci, 3, 3), g, 3)
    b = torch.randn(co, generator=g)
    Ho, Wo = H // stride, W // stride
    if stride == 1:
        acc = torch.nn.functional.conv2d(x.double(), w.double(), padding=1)
    else:
        acc = torch.nn.functional.conv2d(torch.nn.functional.pad(x.double(), (0, 1, 0, 1)), w.double(), stride=2)
    acc = acc.float().permute(0, 2, 3, 1).reshape(-1, co)                  # exact: |sum| < 9 * 192 * 49 units of 2^-5
    pad = 64
    total = n * Ho * Wo * co
    buf = kr.canary_like(1, pad + total + pad, BF16)
    res = torch.randn(n * Ho * Wo, co, generator=g).to(BF16) if with_res else None
    want = buf.clone()
    want[0, pad:pad + total] = (kr.epi_gate_res(acc, b, None, res) if with_res else kr.epi_bias(acc, b)).reshape(-1)
    out = buf.cuda()
    xg = x.permute(0, 2, 3, 1).contiguous().cuda()
    wg = w.permute(0, 2, 3, 1).reshape(co, 9 * ci).contiguous().cuda()
    rg = None if res is None else res.cuda()
    bg = b.cuda()
    _lib.check(_lib.lib().vcb_conv3x3_nhwc(xg.data_ptr(), wg.data_ptr(), bg.data_ptr(), None if rg is None else rg.data_ptr(),
                                           out.data_ptr() + 2 * pad, n, H, W, ci, co, stride, None), "conv")
    torch.cuda.synchronize()
    e = kr.check_exact(out.cpu(), want, f"conv {case}")
    assert e is None, e


@pytest.mark.parametrize("hw", [(7, 16), (16, 9), (1, 2)])
def test_conv3x3_stride2_refuses_odd_input_sizes(ops, hw):
    """stride 2 takes even H and W only (vcb200.h): odd inputs are refused before anything is launched or written"""
    from visualcloze_b200 import _lib
    H, W = hw
    x = torch.zeros(1, H, W, 64, dtype=BF16, device="cuda")
    w = torch.zeros(8, 9 * 64, dtype=BF16, device="cuda")
    out = kr.canary_like(1, 64 + 8 * H * W, BF16).cuda()
    rc = _lib.lib().vcb_conv3x3_nhwc(x.data_ptr(), w.data_ptr(), None, None, out.data_ptr(), 1, H, W, 64, 8, 2, None)
    torch.cuda.synchronize()
    assert rc != 0 and b"even" in _lib.lib().vcb_last_error()
    assert bool(kr.bits(out).eq(kr.CANARY_BF16).all())


# ----------------------------------------------------------------------------------------------
# sequence-parallel head routing: the q/k/v columns of head h go to rank h // (heads / W)'s buffer (local stand-ins here)
# ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cg", [1, 2])
@pytest.mark.parametrize("epi", ["qkv", "linear1"])
def test_gemm_sequence_parallel_routing_contract(ops, epi, cg):
    """every sp_out stand-in is a canary-filled [W * Ltot, 3H / W] buffer: the problem's rows of each owner must hold the QKV
    interval of its heads, every other row its canaries; `out` (unused for q/k/v columns) and out2's margins keep theirs"""
    W_, rank, L, H, K, row_off, Ltot, mlp = 2, 1, 300, 512, 1000, 24, 340, 256
    heads, hw = H // 128, H // 2
    N = 3 * H + (mlp if epi == "linear1" else 0)
    g = torch.Generator().manual_seed(41 + cg)
    a, w = kr.exact_bf16((L, K), g, 2), kr.exact_bf16((N, K), g, 3)
    bias = torch.randn(N, generator=g)
    lin = kr.linear_bf16(kr.exact_acc(a, w, GRAIN), bias)
    qs, ks = (1 + 0.25 * torch.randn(128, generator=g)).to(BF16), (1 + 0.25 * torch.randn(128, generator=g)).to(BF16)
    ang = torch.randn(Ltot, 64, generator=g) * 3
    cos, sin = torch.cos(ang), torch.sin(ang)
    rope = torch.stack([cos, sin], -1).permute(1, 0, 2).contiguous()
    lo, hi = kr.qkv_interval(lin[:, :3 * H], qs, ks, cos[row_off:row_off + L], sin[row_off:row_off + L], H)
    bufs = [kr.canary_like(W_ * Ltot, 3 * hw, BF16).cuda() for _ in range(W_)]
    local = kr.canary_like(Ltot, 3 * H, BF16).cuda()
    cat = kr.canary_like(Ltot, H + mlp + 16, BF16).cuda()
    kw = dict(out2=cat, out2_col_offset=H) if epi == "linear1" else {}
    ops.gemm(a.cuda(), w.cuda(), bias.cuda(), local, epilogue=ops.EPI_LINEAR1 if epi == "linear1" else ops.EPI_QKV, hidden=H,
             q_scale=qs.cuda(), k_scale=ks.cuda(), rope=rope.cuda(), rows_per_batch=L, out_batch_rows=Ltot, out_row_offset=row_off,
             cta_group=cg, sp_out=bufs, sp_row_offset=rank * Ltot, **kw)
    torch.cuda.synchronize()
    r0 = rank * Ltot + row_off
    errs = []
    for owner in range(W_):
        want_lo = kr.canary_like(W_ * Ltot, 3 * hw, BF16)
        want_hi = want_lo.clone()
        region = torch.zeros(want_lo.shape, dtype=torch.bool)
        for reg in range(3):
            src = slice(reg * H + owner * hw, reg * H + (owner + 1) * hw)
            want_lo[r0:r0 + L, reg * hw:(reg + 1) * hw] = lo[:, src]
            want_hi[r0:r0 + L, reg * hw:(reg + 1) * hw] = hi[:, src]
        region[r0:r0 + L] = True
        errs.append(kr.check_interval(bufs[owner].cpu(), want_lo, want_hi, region, f"sp {epi} cg={cg} owner {owner}"))
    errs.append(kr.check_exact(local.cpu(), kr.canary_like(Ltot, 3 * H, BF16), f"sp {epi} cg={cg}: out must stay untouched"))
    if epi == "linear1":
        want_lo = kr.canary_like(Ltot, H + mlp + 16, BF16)
        want_hi = want_lo.clone()
        region = torch.zeros(want_lo.shape, dtype=torch.bool)
        want_lo[row_off:row_off + L, H:H + mlp], want_hi[row_off:row_off + L, H:H + mlp] = kr.gelu_interval(lin[:, 3 * H:])
        region[row_off:row_off + L, H:H + mlp] = True
        errs.append(kr.check_interval(cat.cpu(), want_lo, want_hi, region, f"sp linear1 cg={cg} out2"))
    errs = [e for e in errs if e]
    assert not errs, "\n".join(errs)


# ----------------------------------------------------------------------------------------------
# joint attention
# ----------------------------------------------------------------------------------------------
QA, KA = 1.3, 0.9
BOUND = QA * KA * math.sqrt(128.0) * math.log2(math.e) * 1.03


def _attn_qkv(B, L, heads, seed):
    """[B * L, ld] with the columns permuted inside a wider row: v at 8, k at 8 + H, q at 8 + 2H, NaN in the unused columns;
    q and k rows of RMS QA / KA like after QK-RMSNorm (so BOUND holds for score_bound_log2)"""
    H = heads * 128
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B * L, 3, heads, 128, generator=g)
    for i, s in ((0, QA), (1, KA)):
        x[:, i] = s * x[:, i] / x[:, i].pow(2).mean(-1, keepdim=True).sqrt()
    x = x.to(BF16)
    ld = 3 * H + 16
    qkv = torch.full((B * L, ld), float("nan"), dtype=BF16)
    v_col, k_col, q_col = 8, 8 + H, 8 + 2 * H
    for i, c in ((0, q_col), (1, k_col), (2, v_col)):
        qkv[:, c:c + H] = x[:, i].reshape(B * L, H)
    return qkv, dict(q_col=q_col, k_col=k_col, v_col=v_col), x


def _attn_run(ops, qkv, cols, B, L, heads, seqlens, bounded, schedule):
    H = heads * 128
    ldo = LEFT + H + RIGHT
    buf = kr.canary_like(TOP + B * L + BOTTOM, ldo, BF16)
    out = buf.cuda()
    sl = None if seqlens is None else torch.tensor(seqlens, dtype=torch.int32, device="cuda")
    ops.attention(qkv.cuda(), B, L, heads, out[TOP:TOP + B * L], seqlens=sl, out_col_offset=LEFT,
                  score_bound_log2=BOUND if bounded else 0.0, schedule=schedule, **cols)
    torch.cuda.synchronize()
    return out.cpu(), buf


def _attn_check(got, buf, x, B, L, heads, seqlens, what):
    H = heads * 128
    errs = []
    # margins and columns around the output: canaries
    region = torch.zeros(buf.shape, dtype=torch.bool)
    region[TOP:TOP + B * L, LEFT:LEFT + H] = True
    gb, cb = kr.bits(got), kr.bits(buf)
    if bool((~region & (gb != cb)).any()):
        errs.append(f"{what}: written outside the output region ({int((~region & (gb != cb)).sum())} elements)")
    for b in range(B):
        n = L if seqlens is None else seqlens[b]
        rows = slice(TOP + b * L, TOP + (b + 1) * L)
        pad = gb[rows][n:, LEFT:LEFT + H]
        if bool((pad != 0).any()):
            errs.append(f"{what}: sample {b}: padded query rows must be +0 (bits 0x0000), {int((pad != 0).sum())} are not")
        if n == 0:
            continue
        xs = x[b * L:(b + 1) * L]
        for h in range(heads):
            o, bound = kr.attention_ref(xs[:n, 0, h], xs[:, 1, h], xs[:, 2, h], n)
            e = kr.check_attention(got[rows][:n, LEFT + 128 * h:LEFT + 128 * (h + 1)], o, bound, f"{what} sample {b} head {h}")
            if e:
                errs.append(e)
    return errs


@pytest.mark.parametrize("bounded", [False, True])
@pytest.mark.parametrize("schedule", [1, 2], ids=["per_pair", "persistent"])
@pytest.mark.parametrize("L", [1, 2, 127, 128, 129, 256, 257, 1000])
def test_attention_contract(ops, L, schedule, bounded):
    heads = 3 if L in (2, 128, 257, 1000) else 1
    qkv, cols, x = _attn_qkv(1, L, heads, seed=L)
    got, buf = _attn_run(ops, qkv, cols, 1, L, heads, None, bounded, schedule)
    errs = _attn_check(got, buf, x, 1, L, heads, None, f"L={L} heads={heads} sched={schedule} bounded={bounded}")
    assert not errs, "\n".join(errs)


PADDED = [[300, 129, 1], [128, 0, 257]]
GARBAGE = [float("nan"), float("inf"), float("-inf"), 1e30, -1e30]


@pytest.mark.parametrize("bounded", [False, True])
@pytest.mark.parametrize("seqlens", PADDED, ids=["300-129-1", "128-0-257"])
def test_attention_padded_rows_contract(ops, seqlens, bounded):
    """B = 3, L = 300, right padding.  Valid rows against the fp64 bound, padded output rows +0.  Then the same launch with every
    padded row of Q, K and V overwritten by NaN, +-Inf or +-1e30: the padding carries no meaning (the reference drops those rows
    before attention), so valid rows must equal the zero-padding launch bit for bit and padded rows stay +0."""
    B, L, heads = 3, 300, 2
    qkv, cols, x = _attn_qkv(B, L, heads, seed=sum(seqlens))
    for b, n in enumerate(seqlens):
        qkv[b * L + n:(b + 1) * L, 8:8 + 3 * heads * 128] = 0
        x[b * L + n:(b + 1) * L] = 0
    what = f"padded {seqlens} bounded={bounded}"
    got0, buf = _attn_run(ops, qkv, cols, B, L, heads, seqlens, bounded, 1)
    errs = _attn_check(got0, buf, x, B, L, heads, seqlens, what)
    for val in GARBAGE:
        q2 = qkv.clone()
        for b, n in enumerate(seqlens):
            q2[b * L + n:(b + 1) * L, 8:8 + 3 * heads * 128] = val
        got, _ = _attn_run(ops, q2, cols, B, L, heads, seqlens, bounded, 1)
        e = kr.check_exact(got, got0, f"{what} garbage={val}")
        if e:
            errs.append(e)
    assert not errs, "\n".join(errs)
