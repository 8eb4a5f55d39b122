"""References and checkers for element-by-element kernel tests (CPU only; used by test_kernel_contracts_*.py).

Three tools, each stricter than a rel-L2 bound:

* Exact operands.  bf16 operands drawn from small integers times powers of two (a in {-7..7} 2^-2, w in {-7..7} 2^-3) make every
  partial sum of A W^T an exact fp32 number for the K used here (|sum| < 2^24 units of 2^-5), so the accumulator equals
  ``a.float() @ w.float().T`` whatever the summation order, split-K or stream-K fold.  Everything after it is a chain of single
  fp32 operations on exactly known inputs, emulated here bit for bit in the order include/vcb200.h states.
* Interval emulation for the steps that are not exactly reproducible (GELU's __expf / __fdividef, tanh.approx, the QK-RMSNorm
  rsqrtf of a sum in another order): the chain is evaluated at the ends of an input interval, every step monotone, and the two
  ends are rounded outward to fp32 and then to bf16 the way the final store rounds (to nearest, which is monotone).  The kernel's element must lie in that closed interval.  Each slack is stated where it is used.
* Canaries.  Outputs are views into larger buffers filled with a NaN payload that arithmetic never produces; outside the problem
  region every element must keep it bit for bit, inside none may.
"""
from __future__ import annotations

import math

import torch

BF16 = torch.bfloat16
F32 = torch.float32
F64 = torch.float64

CANARY_BF16 = 0x7FA5                 # quiet-NaN payloads: no arithmetic result has them
CANARY_F32 = 0x7FA5A5A5


# ----------------------------------------------------------------------------------------------
# exact operands
# ----------------------------------------------------------------------------------------------
def exact_bf16(shape, gen: torch.Generator, exp2: int, vmax: int = 7) -> torch.Tensor:
    """integers in [-vmax, vmax] times 2^-exp2, as bf16 (exact)"""
    return (torch.randint(-vmax, vmax + 1, tuple(shape), generator=gen).to(F32) * 2.0 ** -exp2).to(BF16)


def exact_e4m3(shape, gen: torch.Generator, vmax: int = 4) -> torch.Tensor:
    """integers in [-vmax, vmax] as float8_e4m3fn (exact for vmax <= 16)"""
    return torch.randint(-vmax, vmax + 1, tuple(shape), generator=gen).to(F32).to(torch.float8_e4m3fn)


def exact_acc(a: torch.Tensor, w: torch.Tensor, grain: float) -> torch.Tensor:
    """A W^T in fp32, exact: every element of a and w times the other's is a multiple of ``grain``, and |partial sum| < 2^24 grain
    for every summation order (checked), so every fp32 partial sum is exact"""
    a64, w64 = a.to(F64), w.to(F64)
    bound = a64.abs() @ w64.abs().T
    assert (float(bound.max()) if bound.numel() else 0.0) < 2.0 ** 24 * grain, "operands too wide for an exact fp32 accumulator"
    return (a64 @ w64.T).to(F32)


# ----------------------------------------------------------------------------------------------
# bf16 rounding helpers
# ----------------------------------------------------------------------------------------------
def rnd(x: torch.Tensor) -> torch.Tensor:
    """fp32 -> nearest bf16 (ties to even) -> fp32: the kernels' bf16_round / store_bf16x8"""
    return x.to(F32).to(BF16).to(F32)


def _bf16_next_up(x: torch.Tensor) -> torch.Tensor:
    b = x.to(BF16).view(torch.int16).to(torch.int32) & 0xFFFF
    nb = torch.where(b == 0x8000, torch.ones_like(b), torch.where(b < 0x8000, b + 1, b - 1))
    nb = torch.where(nb >= 0x8000, nb - 0x10000, nb)
    return nb.to(torch.int16).view(BF16)


def _bf16_next_down(x: torch.Tensor) -> torch.Tensor:
    return -_bf16_next_up(-x.to(BF16))


def bf16_down(x: torch.Tensor) -> torch.Tensor:
    """largest bf16 <= x (x fp64 or fp32)"""
    x = x.to(F64)
    r = x.to(F32).to(BF16)
    return torch.where(r.to(F64) > x, _bf16_next_down(r), r)


def bf16_up(x: torch.Tensor) -> torch.Tensor:
    """smallest bf16 >= x"""
    x = x.to(F64)
    r = x.to(F32).to(BF16)
    return torch.where(r.to(F64) < x, _bf16_next_up(r), r)


def f32_down(x: torch.Tensor) -> torch.Tensor:
    x = x.to(F64)
    r = x.to(F32)
    return torch.where(r.to(F64) > x, torch.nextafter(r, torch.full_like(r, -math.inf)), r)


def f32_up(x: torch.Tensor) -> torch.Tensor:
    x = x.to(F64)
    r = x.to(F32)
    return torch.where(r.to(F64) < x, torch.nextafter(r, torch.full_like(r, math.inf)), r)


# ----------------------------------------------------------------------------------------------
# GEMM epilogues (include/vcb200.h, enum vcb_epilogue), bit for bit on exact operands
# ----------------------------------------------------------------------------------------------
def scale_acc(acc: torch.Tensor, alpha: float = 0.0) -> torch.Tensor:
    """vcb_gemm_args.alpha: the epilogue sees alpha * acc (one fp32 multiply; 0 and 1 leave acc as it is)"""
    return acc if alpha in (0.0, 1.0) else acc * torch.tensor(alpha, dtype=F32)


def linear_bf16(acc: torch.Tensor, bias: torch.Tensor | None) -> torch.Tensor:
    """bf16(acc + bias): the Linear's output (fp32 values on the bf16 grid)"""
    return rnd(acc if bias is None else acc + bias.to(F32))


def epi_bias(acc, bias) -> torch.Tensor:
    return linear_bf16(acc, bias).to(BF16)


def epi_bias_f32(acc, bias) -> torch.Tensor:
    return acc if bias is None else acc + bias.to(F32)


def epi_gate_res(acc, bias, gate_rows: torch.Tensor | None, res: torch.Tensor) -> torch.Tensor:
    """bf16(res + bf16(gate * bf16(acc + bias))); gate_rows: the gate row of every output row (None = ungated residual)"""
    v = linear_bf16(acc, bias)
    gv = v if gate_rows is None else rnd(gate_rows.to(F32) * v)
    return (res.to(F32) + gv).to(BF16)


def epi_gate_res_fp8(acc, scale, bias, gate_rows, res) -> tuple[torch.Tensor, torch.Tensor]:
    """e4m3 operands: no intermediate rounding, out = bf16(res + gate * (acc * scale + bias)).  The kernel's fp32 expression
    res + gate * v may be contracted to one fma, so both candidates are returned (unfused, fused)."""
    v = (acc.to(F64) * scale.to(F64) + (0.0 if bias is None else bias.to(F64))).to(F32)   # fmaf(acc, sa * sw, bias)
    g = torch.ones_like(v) if gate_rows is None else gate_rows.to(F32)
    unfused = (res.to(F32) + g * v).to(BF16)
    fused = (res.to(F64) + g.to(F64) * v.to(F64)).to(F32).to(BF16)
    return unfused, fused


# --- GELU (torch approximate="tanh"), interval ---------------------------------------------------
_BETA, _KAPPA = 0.7978845608028654, 0.044715


def gelu_interval(x: torch.Tensor, fast: bool = False) -> tuple[torch.Tensor, torch.Tensor]:
    """bf16 interval [lo, hi] holding the kernel's GELU of the fp32 values x (exact inputs).

    gelu_tanh (bf16 operands): x / (1 + E), E = __expf(-2u), u = beta (x + kappa x^3) in fp32.
      * u: four fp32 roundings -> relative slack 2^-21 (4 x 2^-24, doubled);
      * __expf = ex2.approx(x log2 e): relative error 2^-22.5 plus the argument's rounding, |2u log2 e| 2^-24 absolute in the
        exponent, i.e. relative 2^-24 * 2|u| * ln 2 * log2 e; slack 2^-21 + 2^-23 * 2|u|;
      * __fdividef: 2 ulp -> relative slack 2^-21.
    gelu_tanh_fast (e4m3 operands): hx + hx * t, t = tanh.approx(u) with relative error 2^-10.99 -> slack 2^-10 on t, 2^-21 on u.
    Every step is monotone in its input, so the ends of each step's interval map to the ends of the next.  Results below 2^-100
    in magnitude are widened to 0 (flush-to-zero in ex2.approx / __fdividef).  The ends are rounded outward to fp32 and then
    to nearest bf16 like the final store (round to nearest is monotone, so this is tighter than rounding outward to bf16 and
    still holds every possible kernel result)."""
    x = x.to(F64)
    u = _BETA * (x + _KAPPA * x ** 3)
    du = u.abs() * 2.0 ** -21
    if fast:
        t_lo, t_hi = torch.tanh(u - du), torch.tanh(u + du)
        t_lo, t_hi = t_lo - t_lo.abs() * 2.0 ** -10, t_hi + t_hi.abs() * 2.0 ** -10
        hx = 0.5 * x
        c1, c2 = hx * (1 + t_lo), hx * (1 + t_hi)
    else:
        e_lo, e_hi = torch.exp(-2 * (u + du)), torch.exp(-2 * (u - du))       # E decreases with u
        rel = 2.0 ** -21 + 2.0 ** -23 * 2 * (u.abs() + du)
        e_lo, e_hi = e_lo * (1 - rel), e_hi * (1 + rel)
        s_lo, s_hi = 1 / (1 + e_hi) * (1 - 2.0 ** -21), 1 / (1 + e_lo) * (1 + 2.0 ** -21)
        c1, c2 = x * s_lo, x * s_hi
    lo, hi = torch.minimum(c1, c2), torch.maximum(c1, c2)
    tiny = 2.0 ** -100
    small = (lo > -tiny) & (hi < tiny)
    lo = torch.where(small | (lo.abs() < tiny), torch.minimum(lo, torch.zeros_like(lo)) - tiny, lo)
    hi = torch.where(small | (hi.abs() < tiny), torch.maximum(hi, torch.zeros_like(hi)) + tiny, hi)
    # the kernel's fp32 result y lies in [f32_down(lo), f32_up(hi)]; its bf16 store rounds to nearest, which is monotone
    return f32_down(lo).to(BF16), f32_up(hi).to(BF16)


def epi_gelu_interval(acc, bias, fast: bool = False, lin: torch.Tensor | None = None):
    """BIAS_GELU: gelu(bf16(acc + bias)) (bf16 operands) or gelu(acc * scale + bias) (e4m3: pass lin, fast=True)"""
    v = linear_bf16(acc, bias) if lin is None else lin
    return gelu_interval(v, fast)


def gelu_emulated(v: torch.Tensor) -> torch.Tensor:
    """the bf16-operand GELU evaluated in fp32 torch ops (an emulation, not the kernel's exact instructions)"""
    v = v.to(F32)
    inner = torch.tensor(_BETA, dtype=F32) * (v + torch.tensor(_KAPPA, dtype=F32) * v * v * v)
    return (v / (1.0 + torch.exp(-2.0 * inner))).to(BF16)


# --- QKV: bias -> QK-RMSNorm -> scale -> RoPE, interval ----------------------------------------
def qkv_interval(lin: torch.Tensor, q_scale, k_scale, cos, sin, hidden: int, rounded: bool = True):
    """[rows, 3 hidden] Linear outputs (fp32; bf16 values for bf16 operands) -> bf16 intervals of the QKV epilogue.

    q, k (per 128-column head): rrms = rsqrtf(sum(x^2) / 128 + 1e-6) -- the kernel sums in its own order (fmaf over 32 pairs per
    lane, then a quad shuffle sum): relative error <= 128 x 2^-24 = 2^-17 on the sum, 2^-22.9 for rsqrt.approx, 2^-24 for the
    scaling and the eps add: slack 2^-16 on rrms, the one non-exact input.  Then x1 = bf16(x rrms), x2 = bf16(x1 s)
    (layers.py:68-72) and the RoPE pair math.py:112-117 as two fp32 products and one fp32 add; each fp32 op and each rounding is
    monotone in each input, so the extreme results come from the ends of x1 and from the four corners of (x0, x1) for RoPE.
    With ``rounded`` False (e4m3 operands) x1, x2 stay fp32.  v columns: exact (the Linear output).
    cos, sin: [rows, 64] fp32 of the mapped output rows."""
    rows = lin.shape[0]
    heads = hidden // 128
    lo = torch.empty(rows, 3 * hidden, dtype=BF16)
    hi = torch.empty_like(lo)
    r = (lambda t: rnd(t)) if rounded else (lambda t: t)
    v = lin[:, 2 * hidden:].to(F32).to(BF16)
    lo[:, 2 * hidden:], hi[:, 2 * hidden:] = v, v
    for region, sc in ((0, q_scale), (1, k_scale)):
        x = lin[:, region * hidden:(region + 1) * hidden].to(F32).reshape(rows, heads, 128)
        ss = (x.to(F64) ** 2).sum(-1, keepdim=True)
        rr = 1.0 / torch.sqrt(ss / 128 + 1e-6)
        rr_lo, rr_hi = f32_down(rr * (1 - 2.0 ** -16)), f32_up(rr * (1 + 2.0 ** -16))
        a, b = r(x * rr_lo), r(x * rr_hi)
        x1_lo, x1_hi = torch.minimum(a, b), torch.maximum(a, b)
        s = sc.to(F32)
        a, b = r(x1_lo * s), r(x1_hi * s)
        x2_lo, x2_hi = torch.minimum(a, b), torch.maximum(a, b)
        e_lo, e_hi = x2_lo[..., 0::2], x2_hi[..., 0::2]
        o_lo, o_hi = x2_lo[..., 1::2], x2_hi[..., 1::2]
        c, sn = cos.to(F32)[:, None, :], sin.to(F32)[:, None, :]
        outs0, outs1 = [], []
        for x0 in (e_lo, e_hi):
            for x1 in (o_lo, o_hi):
                outs0.append(c * x0 + (-sn) * x1)
                outs1.append(sn * x0 + c * x1)
        y0 = torch.stack(outs0)
        y1 = torch.stack(outs1)
        for k, y in ((0, y0), (1, y1)):
            ylo = y.amin(0).to(BF16)                     # the final bf16 store is round-to-nearest: monotone
            yhi = y.amax(0).to(BF16)
            tgt_lo = lo[:, region * hidden:(region + 1) * hidden].view(rows, heads, 64, 2)
            tgt_hi = hi[:, region * hidden:(region + 1) * hidden].view(rows, heads, 64, 2)
            tgt_lo[..., k] = ylo
            tgt_hi[..., k] = yhi
    return lo, hi


# ----------------------------------------------------------------------------------------------
# canary buffers and checkers
# ----------------------------------------------------------------------------------------------
def canary_like(rows: int, cols: int, dtype, device="cpu") -> torch.Tensor:
    if dtype == BF16:
        return torch.full((rows, cols), CANARY_BF16, dtype=torch.int16, device=device).view(BF16)
    if dtype == F32:
        return torch.full((rows, cols), CANARY_F32, dtype=torch.int32, device=device).view(F32)
    raise ValueError(dtype)


def bits(t: torch.Tensor) -> torch.Tensor:
    t = t.detach().cpu().contiguous()
    return t.view(torch.int16) if t.element_size() == 2 else t.view(torch.int32)


def _where(mask: torch.Tensor, limit: int = 6) -> str:
    idx = mask.nonzero()
    return f"{idx.shape[0]} elements, first at {[tuple(int(v) for v in i) for i in idx[:limit]]}"


def check_exact(got: torch.Tensor, want: torch.Tensor, what: str = "") -> str | None:
    """every element bit for bit (canaries included); None = accepted, else a description of the mismatches"""
    gb, wb = bits(got), bits(want)
    if gb.shape != wb.shape:
        return f"{what}: shape {tuple(gb.shape)} != {tuple(wb.shape)}"
    bad = gb != wb
    if bool(bad.any()):
        i = tuple(int(v) for v in bad.nonzero()[0])
        return (f"{what}: {_where(bad)} differ; at {i}: got {got.detach().cpu()[i].item()!r} (bits {int(gb[i]) & 0xFFFFFFFF:#x}), "
                f"want {want.detach().cpu()[i].item()!r} (bits {int(wb[i]) & 0xFFFFFFFF:#x})")
    return None


def check_interval(got: torch.Tensor, lo: torch.Tensor, hi: torch.Tensor, region: torch.Tensor, what: str = "") -> str | None:
    """inside ``region``: lo <= got <= hi, not NaN; outside: got bit-equal to lo (the expected canaries / exact values there)"""
    gb, lb = bits(got), bits(lo)
    out_bad = (~region) & (gb != lb)
    if bool(out_bad.any()):
        return f"{what}: outside the interval region {_where(out_bad)} differ from the expected bits"
    g, l, h = got.detach().cpu().to(F64), lo.to(F64), hi.to(F64)
    in_bad = region & ~((g >= l) & (g <= h))
    if bool(in_bad.any()):
        i = tuple(int(v) for v in in_bad.nonzero()[0])
        return f"{what}: {_where(in_bad)} outside their interval; at {i}: got {float(g[i])!r} not in [{float(l[i])!r}, {float(h[i])!r}]"
    return None


def check_no_canary(got: torch.Tensor, region: torch.Tensor, what: str = "") -> str | None:
    gb = bits(got)
    c = CANARY_BF16 if gb.dtype == torch.int16 else CANARY_F32
    bad = region & (gb == c)
    return f"{what}: {_where(bad)} inside the problem still hold the canary" if bool(bad.any()) else None


# ----------------------------------------------------------------------------------------------
# attention: fp64 reference and per-element bound
# ----------------------------------------------------------------------------------------------
SCALE = 128 ** -0.5


def attention_ref(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, seqlen: int, scale: float = SCALE):
    """one sample, one head: q/k/v [L, 128] bf16.  Returns (o [seqlen, 128] fp64, bound [seqlen, 128] fp64).

    o = softmax(q k^T scale) v over keys < seqlen, in fp64.  The kernel's rounding points and their worst cases, per query row
    with pi_j = p_j / l the exact probabilities, A = sum_j pi_j |v_j| and n = seqlen keys in T = ceil(n / 128) key tiles:
      1. P rounded to bf16 for the PV product (round to nearest, 8 significant bits, so half an ulp is up to 2^-8 of the value,
         not 2^-9: p = 0.3622 rounds to 0.3613):  <= 2^-8 A.
      2. exponent of p_j: the fp32 score q.k_j (128 exact products summed in fp32, <= 128 x 2^-23 sum_d |q_d k_jd|, 2^-23 rather
         than 2^-24 in case the tensor core truncates), its product with the fp32 constant scale*log2(e) (2 x 2^-24 relative), the
         fma with the row reference (2^-24 |t_j|), ex2.approx (2^-22 relative) and up to T online rescales (ex2 + fp32 multiply,
         2^-22 + 2^-23 each): p_j carries a relative error eta_j <= ln 2 dt_j + (T + 1) 2^-21.  Common factors cancel between O
         and l; what remains is |sum_j pi_j eta_j (v_j - o)| <= sum_j pi_j eta_j (|v_j| + |o|), divided by (1 - max eta).
      3. fp32 sums: l over n unrounded p_j (n 2^-24 relative) and O over n products (n 2^-23 relative to sum p_j |v_j|):
         <= n 2^-22 A.
      4. 1 / l and the product (2 x 2^-24 relative), then the bf16 store: half an ulp of the value stored.
    bound = (2^-8 + n 2^-22 + 2^-22) A + (2) / (1 - max eta) + 1/2 ulp_bf16(|o| + that) + 2^-126 (flush-to-zero in ex2)."""
    n = seqlen
    qf, kf, vf = q.to(F64), k[:n].to(F64), v[:n].to(F64)
    s = (qf @ kf.T) * scale
    m = s.amax(-1, keepdim=True)
    p = torch.exp(s - m)
    l = p.sum(-1, keepdim=True)
    pi = p / l
    o = pi @ vf
    A = pi @ vf.abs()
    T = (n + 127) // 128
    sabs = qf.abs() @ kf.abs().T
    ls2 = scale / math.log(2)                                    # scale in log2 units
    t = (s - m) / math.log(2)
    dt = ls2 * (128 * 2.0 ** -23 * sabs + 2.0 ** -23 * s.abs()) + 2.0 ** -24 * t.abs() + 2.0 ** -24 * (m.abs() / math.log(2))
    eta = math.log(2) * dt + (T + 1) * 2.0 ** -21
    e2 = ((pi * eta) @ vf.abs() + (pi * eta).sum(-1, keepdim=True) * o.abs()) / (1 - eta.amax(-1, keepdim=True))
    pre = (2.0 ** -8 + (n + 1) * 2.0 ** -22) * A + e2
    mag = o.abs() + pre
    ulp = torch.where(mag > 0, 2.0 ** (torch.floor(torch.log2(mag.clamp_min(2.0 ** -133))) - 7), torch.zeros_like(mag))
    bound = pre + 0.5 * ulp + 2.0 ** -126
    return o, bound


def check_attention(got: torch.Tensor, o: torch.Tensor, bound: torch.Tensor, what: str = "") -> str | None:
    """valid query rows of one (sample, head): |got - o| <= bound element by element, no NaN"""
    g = got.detach().cpu().to(F64)
    err = (g - o).abs()
    bad = ~(err <= bound)
    if bool(bad.any()):
        i = tuple(int(x) for x in bad.nonzero()[0])
        return (f"{what}: {_where(bad)} outside the bound; at {i}: got {float(g[i])!r}, ref {float(o[i])!r}, "
                f"|err| {float(err[i]):.3e} > bound {float(bound[i]):.3e}")
    return None


def attention_emulated(q, k, v, seqlen: int, scale: float = SCALE) -> torch.Tensor:
    """fp32 emulation with the kernel's rounding points (fp32 scores, P rounded to bf16 for PV, unrounded row sum, bf16 store)"""
    n = seqlen
    s = (q.to(F32) @ k[:n].to(F32).T) * torch.tensor(scale * math.log2(math.e), dtype=F32)
    m = s.amax(-1, keepdim=True)
    p = torch.exp2(s - m)
    l = p.sum(-1, keepdim=True)
    return ((p.to(BF16).to(F32) @ v[:n].to(F32)) * (1.0 / l)).to(BF16)
