"""Thin torch-tensor wrappers over the C ABI (pointer + size marshalling only; no arithmetic here)."""
from __future__ import annotations

import ctypes as C

import torch

from . import _lib
from ._lib import GemmArgs, check

EPI_BIAS, EPI_BIAS_GELU, EPI_GATE_RES, EPI_QKV, EPI_LINEAR1 = range(5)
BF16 = torch.bfloat16


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


def _p(t: torch.Tensor | None) -> int | None:
    return None if t is None else t.data_ptr()


def _req(t: torch.Tensor, dtype, name: str):
    if not t.is_cuda:
        raise _lib.VcbError(f"{name} must be a CUDA tensor (no CPU fallback)")
    if t.dtype != dtype:
        raise _lib.VcbError(f"{name} must be {dtype}, got {t.dtype}")
    if t.stride(-1) != 1:
        raise _lib.VcbError(f"{name} must be contiguous in its last dimension")


def gemm(*args, **kw) -> torch.Tensor:
    """out[...] = epilogue(a @ w.T); see ``gemm_args`` for the parameters and include/vcb200.h for the semantics."""
    g, out = gemm_args(*args, **kw)
    check(_lib.lib().vcb_gemm_bf16(C.byref(g), _stream()), "vcb_gemm_bf16")
    return out


def gemm_grouped(problem0: dict, problem1: dict) -> None:
    """Two problems (dicts of ``gemm_args`` keyword arguments incl. a, w, bias, out) with equal N, K, epilogue in one launch."""
    def build(d):
        d = dict(d)
        return gemm_args(d.pop("a"), d.pop("w"), d.pop("bias"), d.pop("out"), **d)[0]
    g0, g1 = build(problem0), build(problem1)
    check(_lib.lib().vcb_gemm_bf16_grouped(C.byref(g0), C.byref(g1), _stream()), "vcb_gemm_bf16_grouped")


def gemm_args(a: torch.Tensor, w: torch.Tensor, bias: torch.Tensor | None, out: torch.Tensor, *, epilogue: int = EPI_BIAS,
         out_col_offset: int = 0, rows_per_batch: int | None = None, out_batch_rows: int | None = None,
         out_row_offset: int = 0, gate: torch.Tensor | None = None, res: torch.Tensor | None = None,
         hidden: int = 0, q_scale=None, k_scale=None, rope=None, out2=None, out2_col_offset: int = 0,
         block_n: int = 0, cta_group: int = 0, a_batch_stride: int = 0, m: int | None = None,
         sp_out: list | None = None, sp_row_offset: int = 0, a_scale: torch.Tensor | None = None,
         w_scale: torch.Tensor | None = None, row_stats: torch.Tensor | None = None, lora_t: torch.Tensor | None = None,
         lora_b: torch.Tensor | None = None, lora_t_batch_stride: int = 0, alpha: float = 0.0):
    """out[...] = epilogue(a @ w.T).  a [M,K], w [N,K], out 2-D (rows, ld); see include/vcb200.h.
    With batching (rows_per_batch < M) sample b's rows start at a + b * a_batch_stride (elements).
    fp8: a and w of dtype ``torch.float8_e4m3fn`` (both), with ``a_scale`` [output rows] / ``w_scale`` [N] fp32.
    LoRA k-tail: ``lora_t`` [rows, r] (addressed like ``a``, sample b at lora_t + b * lora_t_batch_stride) and ``lora_b`` [N, r]
    bf16 add ``lora_t @ lora_b.T`` to the accumulator.  ``alpha``: output scale, the epilogue sees alpha * acc (0 = 1)."""
    fp8 = a.dtype == torch.float8_e4m3fn
    if fp8:
        _req(a, torch.float8_e4m3fn, "a"); _req(w, torch.float8_e4m3fn, "w")
    else:
        _req(a, BF16, "a"); _req(w, BF16, "w")
    _req(out, BF16, "out")
    M, K = a.shape
    if m is not None:
        M = m
    N = w.shape[0]
    g = GemmArgs()
    g.M, g.N, g.K = M, N, K
    g.A, g.lda, g.a_batch_stride = a.data_ptr(), a.stride(0), a_batch_stride
    g.W, g.ldw = w.data_ptr(), w.stride(0)
    if bias is not None:
        _req(bias, torch.float32, "bias")
    g.bias = _p(bias)
    g.out, g.ldo, g.out_col_offset = out.data_ptr(), out.stride(0), out_col_offset
    g.rows_per_batch = rows_per_batch or M
    g.out_batch_rows = out_batch_rows if out_batch_rows is not None else g.rows_per_batch
    g.out_row_offset = out_row_offset
    g.epilogue = epilogue
    if gate is not None:
        _req(gate, BF16, "gate")
        g.gate, g.gate_stride = gate.data_ptr(), gate.stride(0)
    if res is not None:                                   # gate None + res: the ungated residual out = bf16(res + bf16(acc + bias))
        _req(res, BF16, "res")
        g.res, g.ld_res = res.data_ptr(), res.stride(0)
    g.hidden = hidden
    g.q_scale, g.k_scale, g.rope = _p(q_scale), _p(k_scale), _p(rope)
    g.rope_rows = 0 if rope is None else rope.shape[1]            # rope is pair-major [64, rows, 2] fp32
    if out2 is not None:
        _req(out2, BF16, "out2")
        g.out2, g.ldo2, g.out2_col_offset = out2.data_ptr(), out2.stride(0), out2_col_offset
    g.block_n, g.cta_group = block_n, cta_group
    if sp_out is not None:
        # sequence-parallel head routing: tensors (local stand-ins in tests) or raw peer-mapped addresses, one per rank
        g.sp_world, g.sp_row_offset = len(sp_out), sp_row_offset
        for r, t in enumerate(sp_out):
            g.sp_out[r] = t.data_ptr() if torch.is_tensor(t) else int(t)
    if row_stats is not None:
        _req(row_stats, torch.float32, "row_stats")          # [output rows, N / 64, 2] fp32 (GATE_RES only)
        g.row_stats = row_stats.data_ptr()
    if fp8:
        g.operand_dtype = 1
        if a_scale is not None:
            _req(a_scale, torch.float32, "a_scale")
        if w_scale is not None:
            _req(w_scale, torch.float32, "w_scale")
        g.a_scale, g.w_scale = _p(a_scale), _p(w_scale)
    if lora_t is not None or lora_b is not None:
        _req(lora_t, BF16, "lora_t"); _req(lora_b, BF16, "lora_b")
        if lora_b.stride(0) != lora_b.shape[1]:
            raise _lib.VcbError("lora_b must be a dense [N, r] matrix")
        g.lora_t, g.ld_lora_t, g.lora_t_batch_stride = lora_t.data_ptr(), lora_t.stride(0), lora_t_batch_stride
        g.lora_b, g.lora_rank = lora_b.data_ptr(), lora_b.shape[1]
    g.alpha = alpha
    g._keepalive = (a, w, bias, out, gate, res, q_scale, k_scale, rope, out2, sp_out, a_scale, w_scale, row_stats, lora_t, lora_b)
    return g, out


def attention(qkv: torch.Tensor, B: int, L: int, heads: int, out: torch.Tensor, *, q_col: int, k_col: int, v_col: int,
              seqlens: torch.Tensor | None = None, out_col_offset: int = 0, score_bound_log2: float = 0.0,
              schedule: int = 0) -> torch.Tensor:
    """qkv [B*L, ld] bf16 (post RoPE / QK-norm) -> out [B*L, ldo]; models/math.py:63-99.
    ``score_bound_log2`` > 0: promised bound of the scaled scores (vcb_attn_args) -> softmax without a running row max."""
    _req(qkv, BF16, "qkv"); _req(out, BF16, "out")
    if seqlens is not None:
        _req(seqlens, torch.int32, "seqlens")
    if score_bound_log2 or schedule:
        a = _lib.AttnArgs()
        a.schedule = int(schedule)
        a.qkv, a.ld_qkv, a.q_col, a.k_col, a.v_col = qkv.data_ptr(), qkv.stride(0), q_col, k_col, v_col
        a.seqlens, a.B, a.L, a.heads = _p(seqlens), B, L, heads
        a.out, a.ldo, a.out_col_offset, a.score_bound_log2 = out.data_ptr(), out.stride(0), out_col_offset, float(score_bound_log2)
        check(_lib.lib().vcb_attention_fwd_ex(C.byref(a), _stream()), "vcb_attention_fwd_ex")
        return out
    check(_lib.lib().vcb_attention_fwd(qkv.data_ptr(), qkv.stride(0), q_col, k_col, v_col, _p(seqlens), B, L, heads,
                                       out.data_ptr(), out.stride(0), out_col_offset, _stream()), "vcb_attention_fwd")
    return out


def attention_sp(qkv: torch.Tensor, L: int, heads: int, out_peers: list, rows_per_rank: int, ldo: int, *, q_col: int, k_col: int,
                 v_col: int, out_col_offset: int = 0) -> None:
    """Sequence-parallel attention of this rank's ``heads`` heads over all L rows; query row r is stored into
    ``out_peers[r // rows_per_rank]`` (tensors or raw peer-mapped addresses, leading dimension ``ldo``) at row r % rows_per_rank."""
    _req(qkv, BF16, "qkv")
    arr = (C.c_void_p * len(out_peers))(*[(t.data_ptr() if torch.is_tensor(t) else int(t)) for t in out_peers])
    check(_lib.lib().vcb_attention_fwd_sp(qkv.data_ptr(), qkv.stride(0), q_col, k_col, v_col, L, heads, arr, len(out_peers),
                                          rows_per_rank, ldo, out_col_offset, _stream()), "vcb_attention_fwd_sp")


def ln_modulate(x: torch.Tensor, shift: torch.Tensor, scale: torch.Tensor, out: torch.Tensor, rows_per_batch: int,
                mod_stride: int | None = None, rows: int | None = None, batch_rows: int = 0) -> torch.Tensor:
    """out = bf16((1 + scale[b]) * LayerNorm(x) + shift[b]); x/out [rows, H]; shift/scale rows per sample."""
    _req(x, BF16, "x"); _req(out, BF16, "out"); _req(shift, BF16, "shift"); _req(scale, BF16, "scale")
    H = x.shape[1]
    rows = rows if rows is not None else x.shape[0]
    ms = mod_stride if mod_stride is not None else (shift.stride(0) if shift.dim() > 1 else 0)
    check(_lib.lib().vcb_ln_modulate(x.data_ptr(), x.stride(0), out.data_ptr(), out.stride(0), shift.data_ptr(),
                                     scale.data_ptr(), ms, rows, H, rows_per_batch, batch_rows, _stream()), "vcb_ln_modulate")
    return out


def _ln_launch(x: torch.Tensor, out: torch.Tensor, problems: list, hidden: int, batch_rows: int, mod_stride: int,
               row_scale: torch.Tensor | None = None, stats: torch.Tensor | None = None) -> None:
    """One AdaLN LayerNorm launch over one or two problems (row_offset, rows, rows_per_batch, shift, scale) of the [*, hidden]
    buffers x / out: out bf16, or float8_e4m3fn with ``row_scale`` [*] fp32; ``stats`` [*, n_slots, 2] fp32: row statistics
    supplied by the producing GEMM.  row_scale and stats are indexed by the row of x, like out."""
    fp8 = out.dtype == torch.float8_e4m3fn
    _req(x, BF16, "x"); _req(out, torch.float8_e4m3fn if fp8 else BF16, "out")
    if fp8:
        _req(row_scale, torch.float32, "row_scale")
    if stats is not None:
        _req(stats, torch.float32, "stats")
    args, rs, st = [None, None], [None, None], [None, None]
    for i, (off, rows, rpb, shift, scale) in enumerate(problems):
        _req(shift, BF16, "shift"); _req(scale, BF16, "scale")
        a = _lib.LnArgs()
        a.x, a.y = x.data_ptr() + off * x.stride(0) * 2, out.data_ptr() + off * out.stride(0) * out.element_size()
        a.shift, a.scale, a.rows, a.rows_per_batch = shift.data_ptr(), scale.data_ptr(), rows, rpb
        args[i] = C.byref(a)
        if fp8:
            rs[i] = row_scale.data_ptr() + off * 4
        if stats is not None:
            st[i] = stats.data_ptr() + off * stats.stride(0) * 4
    common = (x.stride(0), out.stride(0), mod_stride, hidden, batch_rows, _stream())
    lib = _lib.lib()
    if stats is not None and fp8:
        check(lib.vcb_ln_modulate_fp8_stats(*args, *rs, *st, stats.shape[1], *common), "vcb_ln_modulate_fp8_stats")
    elif stats is not None:
        check(lib.vcb_ln_modulate_stats(*args, *st, stats.shape[1], *common), "vcb_ln_modulate_stats")
    elif fp8:
        check(lib.vcb_ln_modulate_fp8(*args, *rs, *common), "vcb_ln_modulate_fp8")
    else:
        check(lib.vcb_ln_modulate_grouped(*args, *common), "vcb_ln_modulate_grouped")


def ln_modulate_grouped(x: torch.Tensor, out: torch.Tensor, problems: list, hidden: int, batch_rows: int, mod_stride: int, *,
                        row_scale: torch.Tensor | None = None, stats: torch.Tensor | None = None) -> None:
    """Two row ranges of the joint buffers in one launch.  ``problems``: two (or one) tuples (row_offset, rows, rows_per_batch, shift,
    scale); x / out are the [*, hidden] joint buffers.  out float8_e4m3fn with ``row_scale``: the e4m3 form; ``stats``: row
    statistics supplied by the producing GEMM (see ``_ln_launch``)."""
    _ln_launch(x, out, problems, hidden, batch_rows, mod_stride, row_scale, stats)


def ln_modulate_stats(x: torch.Tensor, shift: torch.Tensor, scale: torch.Tensor, out: torch.Tensor, stats: torch.Tensor,
                      rows_per_batch: int, mod_stride: int | None = None, batch_rows: int | None = None) -> torch.Tensor:
    """``ln_modulate`` with the row statistics supplied by the producing GEMM: stats [rows, n_slots, 2] fp32 (sum, sum of squares)."""
    ms = mod_stride if mod_stride is not None else (shift.stride(0) if shift.dim() > 1 else 0)
    _ln_launch(x, out, [(0, x.shape[0], rows_per_batch, shift, scale)], x.shape[1], batch_rows or rows_per_batch, ms, stats=stats)
    return out


def quantize_rows_e4m3(x: torch.Tensor, out8: torch.Tensor, row_scale: torch.Tensor) -> None:
    """x [rows, K] bf16 (any row stride) -> out8 [rows, K] float8_e4m3fn and row_scale [rows] fp32 = max(max|x|, 1e-12) / 448
    (x ~= out8 * row_scale): the activation side of the fp8 Linears that are not fed by a LayerNorm (vcb_quantize_rows_e4m3)."""
    rows, K = x.shape
    assert x.dtype == torch.bfloat16 and out8.dtype == torch.float8_e4m3fn and row_scale.dtype == torch.float32
    assert out8.shape == x.shape and row_scale.numel() == rows and x.stride(1) == 1 and out8.stride(1) == 1
    check(_lib.lib().vcb_quantize_rows_e4m3(x.data_ptr(), x.stride(0), out8.data_ptr(), out8.stride(0), row_scale.data_ptr(), rows, K,
                                            _stream()), "vcb_quantize_rows_e4m3")


def ln_modulate_fp8(x: torch.Tensor, shift: torch.Tensor, scale: torch.Tensor, out8: torch.Tensor, row_scale: torch.Tensor,
                    rows_per_batch: int, mod_stride: int | None = None, batch_rows: int | None = None,
                    stats: torch.Tensor | None = None) -> torch.Tensor:
    """e4m3 form of ``ln_modulate``: out8 [rows, H] float8_e4m3fn, row_scale [rows] fp32 (max|y| / 448 per row).
    ``stats`` [rows, n_slots, 2] fp32: row statistics supplied by the producing GEMM (vcb_ln_modulate_fp8_stats)."""
    ms = mod_stride if mod_stride is not None else (shift.stride(0) if shift.dim() > 1 else 0)
    _ln_launch(x, out8, [(0, x.shape[0], rows_per_batch, shift, scale)], x.shape[1], batch_rows or rows_per_batch, ms, row_scale, stats)
    return out8


# ---- text encoders (models/modules/conditioner.py:5-37; include/vcb200.h "text encoders") -----------------------------------
def embedding(table: torch.Tensor, ids: torch.Tensor, out: torch.Tensor, pos_table: torch.Tensor | None = None, L: int = 0) -> torch.Tensor:
    """out[t] = table[ids[t]] (+ pos_table[t % L]); table [vocab, dim] bf16, ids int64 [n], out [n, dim] bf16"""
    _req(table, BF16, "table"); _req(out, BF16, "out"); _req(ids, torch.int64, "ids")
    check(_lib.lib().vcb_embedding_bf16(table.data_ptr(), table.shape[0], table.shape[1], ids.data_ptr(), _p(pos_table), L, out.data_ptr(),
                                        out.stride(0), ids.numel(), _stream()), "vcb_embedding_bf16")
    return out


def rmsnorm_weight(x: torch.Tensor, weight: torch.Tensor, out: torch.Tensor, eps: float) -> torch.Tensor:
    """T5LayerNorm: out = weight * bf16(x * rsqrt(mean(x^2) + eps)); x / out [rows, dim] bf16"""
    _req(x, BF16, "x"); _req(weight, BF16, "weight"); _req(out, BF16, "out")
    check(_lib.lib().vcb_rmsnorm_weight(x.data_ptr(), x.stride(0), weight.data_ptr(), out.data_ptr(), out.stride(0), x.shape[0], x.shape[1],
                                        float(eps), _stream()), "vcb_rmsnorm_weight")
    return out


def layernorm_affine(x: torch.Tensor, weight: torch.Tensor, bias: torch.Tensor, out: torch.Tensor, eps: float) -> torch.Tensor:
    _req(x, BF16, "x"); _req(weight, BF16, "weight"); _req(bias, BF16, "bias"); _req(out, BF16, "out")
    check(_lib.lib().vcb_layernorm_affine(x.data_ptr(), x.stride(0), weight.data_ptr(), bias.data_ptr(), out.data_ptr(), out.stride(0),
                                          x.shape[0], x.shape[1], float(eps), _stream()), "vcb_layernorm_affine")
    return out


def gated_gelu(ab: torch.Tensor, out: torch.Tensor) -> torch.Tensor:
    """out = gelu_new(ab[:, :dff]) * ab[:, dff:]; ab [rows, 2 * dff], out [rows, dff]"""
    _req(ab, BF16, "ab"); _req(out, BF16, "out")
    check(_lib.lib().vcb_gated_gelu(ab.data_ptr(), ab.stride(0), out.data_ptr(), out.stride(0), ab.shape[0], out.shape[1], _stream()),
          "vcb_gated_gelu")
    return out


def quick_gelu(x: torch.Tensor, out: torch.Tensor) -> torch.Tensor:
    _req(x, BF16, "x"); _req(out, BF16, "out")
    check(_lib.lib().vcb_quick_gelu(x.data_ptr(), out.data_ptr(), x.numel(), _stream()), "vcb_quick_gelu")
    return out


def attention_small(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, out: torch.Tensor, B: int, L: int, heads: int, *,
                    bias: torch.Tensor | None = None, scale: float = 1.0, causal: bool = False) -> torch.Tensor:
    """head_dim-64 attention of the text encoders; q / k / v: 2-D views [B * L, heads * 64] (may be column windows of one fused
    buffer, equal row strides); bias [heads, L, L] bf16 or None"""
    for t, n in ((q, "q"), (k, "k"), (v, "v"), (out, "out")):
        _req(t, BF16, n)
    assert q.stride(0) == k.stride(0) == v.stride(0)
    a = _lib.AttnSmallArgs()
    a.q, a.k, a.v, a.ld = q.data_ptr(), k.data_ptr(), v.data_ptr(), q.stride(0)
    if bias is not None:
        _req(bias, BF16, "bias")
        assert tuple(bias.shape) == (heads, L, L) and bias.is_contiguous()
    a.bias = _p(bias)
    a.out, a.ldo = out.data_ptr(), out.stride(0)
    a.B, a.L, a.heads, a.head_dim, a.causal, a.scale = B, L, heads, 64, int(causal), float(scale)
    a._keepalive = (q, k, v, out, bias)
    check(_lib.lib().vcb_attention_small(C.byref(a), _stream()), "vcb_attention_small")
    return out


def timestep_embedding(t_scaled: torch.Tensor, freqs: torch.Tensor, out: torch.Tensor) -> torch.Tensor:
    _req(t_scaled, torch.float32, "t_scaled"); _req(freqs, torch.float32, "freqs"); _req(out, BF16, "out")
    check(_lib.lib().vcb_timestep_embedding(t_scaled.data_ptr(), freqs.data_ptr(), out.data_ptr(), t_scaled.numel(),
                                            _stream()), "vcb_timestep_embedding")
    return out


def silu(x: torch.Tensor, out: torch.Tensor) -> torch.Tensor:
    _req(x, BF16, "x"); _req(out, BF16, "out")
    check(_lib.lib().vcb_silu(x.data_ptr(), out.data_ptr(), x.numel(), _stream()), "vcb_silu")
    return out


def add3(a, b, c, out) -> torch.Tensor:
    _req(a, BF16, "a"); _req(out, BF16, "out")
    rows, H = a.shape
    check(_lib.lib().vcb_add3(a.data_ptr(), _p(b), 0 if b is None else b.shape[0], _p(c), 0 if c is None else c.shape[0],
                              out.data_ptr(), rows, H, _stream()), "vcb_add3")
    return out


def rope_table(ids: torch.Tensor, axes_dim, theta: float, out: torch.Tensor) -> torch.Tensor:
    """ids [rows, 3] fp32 -> out [64, rows, 2] fp32 (cos, sin), pair-major."""
    _req(ids, torch.float32, "ids"); _req(out, torch.float32, "out")
    check(_lib.lib().vcb_rope_table(ids.data_ptr(), out.data_ptr(), ids.shape[0], axes_dim[0], axes_dim[1], axes_dim[2],
                                    float(theta), _stream()), "vcb_rope_table")
    return out


def euler_update(x, v, dt_bf16: float, x_new, model_in=None) -> torch.Tensor:
    """x_new = bf16(x + bf16(dt * (-v))) on dense [rows, C] matrices (the kernel indexes x, v and x_new flat)."""
    _req(x, BF16, "x"); _req(v, BF16, "v"); _req(x_new, BF16, "x_new")
    rows, Cc = x.shape
    if not v.is_contiguous():
        v = v.contiguous()                   # e.g. a foreign model returning a column slice y[..., :64]
    for name, t in (("x", x), ("v", v), ("x_new", x_new)):
        if tuple(t.shape) != (rows, Cc) or t.stride(0) != Cc:
            raise ValueError(f"euler_update: {name} must be a dense [{rows}, {Cc}] matrix, got shape {tuple(t.shape)} strides {t.stride()}")
    check(_lib.lib().vcb_euler_update(x.data_ptr(), v.data_ptr(), dt_bf16, x_new.data_ptr(), _p(model_in),
                                      0 if model_in is None else model_in.stride(0), rows, Cc, _stream()),
          "vcb_euler_update")
    return x_new


ODE_METHODS = {"euler": 0, "midpoint": 1, "rk4": 2}          # VCB_ODE_* (include/vcb200.h)
ODE_STAGES = {"euler": 1, "midpoint": 2, "rk4": 4}           # model evaluations per interval


def ode_stage(method: str, stage: int, y0, vs, dt: float, y_out, model_in=None) -> torch.Tensor:
    """One stage update of a fixed-grid solver (``vcb_ode_stage``): ``vs`` are the model outputs v_1..v_{stage+1} of the interval,
    ``dt`` the fp32 ``t1 - t0``; writes y_out and, if given, columns [0, C) of model_in.  See include/vcb200.h for the expressions."""
    if method not in ODE_METHODS:
        raise ValueError(f"ode_stage: method must be one of {sorted(ODE_METHODS)}, got {method!r}")
    _req(y0, BF16, "y0"); _req(y_out, BF16, "y_out")
    rows, Cc = y0.shape
    vs = [v if v.is_contiguous() else v.contiguous() for v in vs]      # e.g. a foreign model returning a column slice
    for name, t in [("y0", y0), ("y_out", y_out)] + [(f"v[{i}]", v) for i, v in enumerate(vs)]:
        _req(t, BF16, name)
        if tuple(t.shape) != (rows, Cc) or t.stride(0) != Cc:
            raise ValueError(f"ode_stage: {name} must be a dense [{rows}, {Cc}] matrix, got shape {tuple(t.shape)} strides {t.stride()}")
    if model_in is not None:
        _req(model_in, BF16, "model_in")
        if model_in.shape[0] != rows or model_in.shape[1] < Cc:
            raise ValueError(f"ode_stage: model_in must be [{rows}, >= {Cc}], got {tuple(model_in.shape)}")
    ptrs = (C.c_void_p * max(1, len(vs)))(*[v.data_ptr() for v in vs])
    check(_lib.lib().vcb_ode_stage(ODE_METHODS[method], stage, y0.data_ptr(), ptrs, len(vs), dt, y_out.data_ptr(),
                                   _p(model_in), 0 if model_in is None else model_in.stride(0), rows, Cc, _stream()),
          "vcb_ode_stage")
    return y_out


def copy_cols(src, dst, col0: int) -> torch.Tensor:
    _req(src, BF16, "src"); _req(dst, BF16, "dst")
    rows, Cc = src.shape
    check(_lib.lib().vcb_copy_cols(src.data_ptr(), src.stride(0), dst.data_ptr(), dst.stride(0), col0, rows, Cc,
                                   _stream()), "vcb_copy_cols")
    return dst


def umma_probe(a, b, ksteps: int, b_mn_major: bool, a_from_regs: bool, b_lbo: int = 0, b_sbo: int = 0,
               b_kstep_bytes: int = 0) -> torch.Tensor:
    out = torch.empty(128, 128, dtype=torch.float32, device=a.device)
    check(_lib.lib().vcb_debug_umma_probe(a.data_ptr(), b.data_ptr(), out.data_ptr(), ksteps, int(b_mn_major),
                                          int(a_from_regs), b_lbo, b_sbo, b_kstep_bytes, _stream()), "vcb_debug_umma_probe")
    return out
