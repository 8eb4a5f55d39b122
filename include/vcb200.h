/* vcb200.h -- C ABI of libvcb200.so: the H100-native (sm_90a) VisualCloze denoising hot path.
 *
 * The reference (lzyhha/VisualCloze) is pure Python and has no FFI layer; its boundary for this path is a set
 * of Python call signatures (SURVEY.md 8b).  Each entry point below names the reference code it replaces
 * (file:line under the reference tree).  The Python mirror of the reference interface
 * (visualcloze_b200/model.py, sampling.py, transport.py, pipeline.py) binds these symbols with ctypes; the
 * binding a reference maintainer would add is shown in INTEGRATION.md.
 *
 * Conventions
 *   - all pointers are DEVICE pointers unless named host_*; the caller owns every buffer;
 *   - bf16 tensors are passed as void* / uint16 storage, row-major, leading dimensions in ELEMENTS;
 *   - `stream` is a cudaStream_t passed as void* (0 = legacy default stream); work is only enqueued;
 *   - every function returns 0 on success, non-zero on error; vcb_last_error() gives the message
 *     (thread-local).  No C++ exception crosses the boundary.  No CPU fallback exists.
 */
#ifndef VCB200_H_
#define VCB200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define VCB_ABI_VERSION 7
#define VCB_SP_MAX 8          /* ranks of one sequence-parallel group (one NVSwitch domain) */

/* ---- library ------------------------------------------------------------------------------ */
int         vcb_abi_version(void);
const char* vcb_last_error(void);
/* number of kernels this library has launched since load / since the last reset (bench.py gpu_launches) */
long long   vcb_launch_count(void);
void        vcb_reset_launch_count(void);
/* Device time per kernel category, measured with CUDA events around every launch between begin and end
 * (categories: 0 GEMM, 1 attention, 2 AdaLN LayerNorm, 3 other).  end synchronises the device.
 * For measurement runs only; not to be used while a CUDA graph is being captured. */
int         vcb_profile_begin(void);
int         vcb_profile_end(double ms[4], long long launches[4]);
/* Extended form: ncat in [4, 6] categories (4 = VAE 3x3 convolutions, 5 = VAE GroupNorm / upsample / softmax / layout; with
 * ncat == 4 they fold into "other"), and optionally one record per launch in launch order.
 * info: GEMM {M, N, K, epilogue | (block_n / 32) << 8 | cta_group << 16 | issued-by-the-VAE-engine << 24}; conv {output pixels, cout, 9 * cin, stride};
 * attention {B, L, heads, fixed-reference softmax | persistent schedule << 1}. */
typedef struct vcb_prof_record { int32_t category; float ms; int32_t info[4]; } vcb_prof_record;
int         vcb_profile_end_ex(double* ms, long long* launches, int32_t ncat, vcb_prof_record* records, int64_t capacity,
                               int64_t* n_records);

/* ---- fused-epilogue GEMM:  D = epilogue(A[M,K] * W[N,K]^T)   (bf16 x bf16 -> fp32 -> bf16) --------------
 * Replaces every nn.Linear on the path (models/modules/layers.py:165,172,190-195,235,244; model.py:101,108;
 * lora.py:92-98 with merged weights, or unmerged through the LoRA k-tail below) together with the elementwise ops that
 * follow it in the reference. */
enum vcb_epilogue {
    VCB_EPI_BIAS = 0,      /* out = bf16(acc + bias) */
    VCB_EPI_BIAS_GELU = 1, /* out = bf16(gelu_tanh(bf16(acc + bias)))                    layers.py:143,154 */
    VCB_EPI_GATE_RES = 2,  /* out = bf16(res + bf16(gate * bf16(acc + bias)))             layers.py:190-195,245 */
    VCB_EPI_QKV = 3,       /* bias; q,k: RMSNorm(128) * scale then RoPE; v: bias only     layers.py:165-174, math.py:112-117 */
    VCB_EPI_LINEAR1 = 4,   /* cols < 3H as QKV -> out; cols >= 3H as BIAS_GELU -> out2     layers.py:235-244 */
    VCB_EPI_BIAS_F32 = 5   /* out is FP32 [.., ldo]: acc + bias (VAE attention scores, autoencoder.py:47) */
};
/* VCB_EPI_GATE_RES with gate == NULL is the ungated residual out = bf16(res + bf16(acc + bias)). */

typedef struct vcb_gemm_args {
    int32_t M, N, K;
    const void* A;  int64_t lda;     /* [M, K] bf16; with batching: sample b starts at A + b * a_batch_stride */
    int64_t a_batch_stride;          /* elements; 0 = rows_per_batch * lda (plain matrix) */
    const void* W;  int64_t ldw;     /* [N, K] bf16 (nn.Linear.weight layout) */
    const float* bias;               /* [N] fp32 or NULL */
    void* out;      int64_t ldo;     /* bf16 */
    int32_t out_col_offset;
    /* batching: M = batch * rows_per_batch; row i of sample b is read from A + b * a_batch_stride + i * lda and
       written to output row b * out_batch_rows + out_row_offset + i (res is indexed the same way, gate by b).
       Set rows_per_batch = M, out_batch_rows = M, out_row_offset = 0 for a plain matrix. */
    int32_t rows_per_batch, out_batch_rows, out_row_offset;
    int32_t epilogue;                /* enum vcb_epilogue */
    /* VCB_EPI_GATE_RES */
    const void* gate; int64_t gate_stride;   /* [B, gate_stride] bf16 */
    const void* res;  int64_t ld_res;        /* bf16, indexed by OUTPUT row; may alias out */
    /* VCB_EPI_QKV / VCB_EPI_LINEAR1 (head_dim is 128) */
    int32_t hidden;
    const void* q_scale; const void* k_scale;   /* [128] bf16 */
    const void* rope;                            /* pair-major [64][rope_rows] float2 (cos, sin); row = mapped output row */
    int64_t rope_rows;
    void* out2; int64_t ldo2; int32_t out2_col_offset;
    /* tuning: 0 = library heuristic */
    int32_t block_n;                 /* 64 / 128 / 192 / 256 */
    int32_t cta_group;               /* 1 or 2 (2-CTA cluster on a 256-row tile, multicast B) */
    /* sequence-parallel head routing (VCB_EPI_QKV / VCB_EPI_LINEAR1, one sample; sp_world <= 1 = off): token rows are
       sharded over sp_world ranks and attention heads over the same ranks, so the epilogue stores the q/k/v columns of
       head h directly into rank h / (heads / sp_world)'s peer-mapped buffer sp_out[rank] -- layout
       [sp_world * rows, 3 * hidden / sp_world], row sp_row_offset + mapped output row -- over NVLink (fused all-to-all).
       `out` is then unused for the q/k/v columns. */
    int32_t sp_world, sp_row_offset;
    void* sp_out[VCB_SP_MAX];
    /* VCB_EPI_GATE_RES, optional: row_stats [output rows][N / 64] float2 -- per row and per 64 output columns the (sum, sum of
       squares) of the bf16 values this GEMM stores, i.e. the statistics the AdaLN LayerNorm that follows needs
       (vcb_ln_modulate_stats); N % 64 == 0, plain matrices, block_n 128 or 256.  NULL = not produced. */
    void* row_stats;
    /* FP8 operands (opt-in; VCB_EPI_BIAS / BIAS_GELU / QKV / LINEAR1, plain matrices): operand_dtype = VCB_DTYPE_E4M3 makes A
       and W e4m3 bytes (lda / ldw / a_batch_stride in elements = bytes, multiples of 16), multiplied on the tensor cores with
       wgmma e4m3 x e4m3; the fp32 accumulator is rescaled by a_scale[mapped OUTPUT row] * w_scale[column] before the
       bias (per-row activation scales as written by vcb_ln_modulate_fp8, per-output-channel weight scales; NULL = 1). */
    int32_t operand_dtype;           /* VCB_DTYPE_BF16 (0) or VCB_DTYPE_E4M3 (1) */
    const float* a_scale;
    const float* w_scale;
    /* Unmerged LoRA k-tail (bf16 operands only; lora_rank 0 = none): out = epilogue(A W^T + T lora_b^T), one fp32 accumulator,
       i.e. [A | T] [W | lora_b]^T.  T [M, lora_rank] bf16 is addressed like A: row i of sample b at
       lora_t + b * lora_t_batch_stride + i * ld_lora_t (batch stride 0 = rows_per_batch * ld_lora_t).  lora_b [N, lora_rank] bf16
       (row stride lora_rank, lora.py's lora_B.weight).  lora_rank % 8 == 0 (the last partial k-block is zero-filled); both problems
       of a grouped launch need the same rank. */
    const void* lora_t; int64_t ld_lora_t;
    int64_t lora_t_batch_stride;
    const void* lora_b;
    int32_t lora_rank;
    /* output scale: the epilogue sees alpha * acc in place of acc (0 = 1).  The LoRA down-projection T = bf16(s * X lora_a^T). */
    float alpha;
} vcb_gemm_args;
#define VCB_DTYPE_BF16 0
#define VCB_DTYPE_E4M3 1

int vcb_gemm_bf16(const vcb_gemm_args* args, void* stream);
/* Two problems with the same N, K and epilogue (their own A, W, bias, outputs, row mapping) in ONE persistent launch:
 * the txt stream of a DoubleStreamBlock (layers.py:170-175,193-195) rides in the img stream's launch and fills its
 * partial last wave.  block_n / cta_group are taken from the first problem. */
int vcb_gemm_bf16_grouped(const vcb_gemm_args* args0, const vcb_gemm_args* args1, void* stream);

/* ---- 3x3 convolution, stride 1, zero padding 1, NHWC bf16 (models/modules/autoencoder.py:63,65,101,239,258) ------
 * Implicit GEMM on the wgmma kernel without im2col: each k-block is one 4-D TMA box of a 16x8 pixel patch at the
 * filter tap's shift, zero-filled outside the image.  x [n,H,W,cin], w [cout, 3,3,cin] (tap-major, channels last),
 * out [n,H/stride,W/stride,cout]; res (optional, same shape as out): out = bf16(res + bf16(conv + bias)).
 * stride 1: zero padding 1 all round.  stride 2: the encoder's Downsample (autoencoder.py:85-95): pad right/bottom by 1,
 * no padding left/top; the TMA map carries elementStrides = 2.  cin % 64 == 0, cout % 8 == 0. */
int vcb_conv3x3_nhwc(const void* x, const void* w, const float* bias, const void* res, void* out, int32_t n,
                     int32_t H, int32_t W, int32_t cin, int32_t cout, int32_t stride, void* stream);

/* ---- joint attention (models/math.py:63-99: attention/_upad_input/flash_attn_varlen_func/pad_input) ------
 * qkv: [B, L, ld_qkv] bf16, head h of q/k/v at columns {q,k,v}_col + 128*h, RoPE + QK-norm already applied.
 * seqlens: [B] int32 valid tokens (right padding) or NULL.  out rows >= seqlen are written as zeros. */
int vcb_attention_fwd(const void* qkv, int64_t ld_qkv, int32_t q_col, int32_t k_col, int32_t v_col,
                      const int32_t* seqlens, int32_t B, int32_t L, int32_t heads,
                      void* out, int64_t ldo, int32_t out_col_offset, void* stream);

/* Sequence-parallel variant (SURVEY.md 8f-2; one sample, no padding): this rank attends `heads` heads over the L rows of
 * ALL ranks held in its qkv buffer and stores query row r into out_peers[r / rows_per_rank] (peer-mapped, row
 * r % rows_per_rank, columns out_col_offset + 128*h) over NVLink -- the return all-to-all fused into the epilogue. */
int vcb_attention_fwd_sp(const void* qkv, int64_t ld_qkv, int32_t q_col, int32_t k_col, int32_t v_col, int32_t L,
                         int32_t heads, void* const* out_peers, int32_t world, int32_t rows_per_rank, int64_t ldo,
                         int32_t out_col_offset, void* stream);

/* General form.  score_bound_log2 > 0 promises |q.k| * 128^-0.5 * log2(e) <= score_bound_log2 for every query/key pair (true
 * after QK-RMSNorm: |q| <= max|q_scale| * sqrt(128), layers.py:63-84): softmax is shift invariant, so the kernel then uses
 * exp2(s - bound) with no running row max -- same result up to rounding, shorter dependency chain.  Must be <= 64 (fp32 /
 * bf16 exponent range); 0 = exact online softmax.  out_peers != NULL selects the sequence-parallel output routing.
 * schedule: PER_PAIR = one CTA per (256-query pair, head, sample); PERSISTENT = one CTA per SM, full rounds dealt like the per-pair
 * grid and the partial last round cut along the key tiles (cut units are folded from fp32 partials; unpadded batches only);
 * AUTO = PER_PAIR unless the environment sets VCB_ATTN_PERSIST=1 (measured: faster alone, equal inside the power-capped loop). */
#define VCB_ATTN_SCHED_AUTO 0
#define VCB_ATTN_SCHED_PER_PAIR 1
#define VCB_ATTN_SCHED_PERSISTENT 2
typedef struct vcb_attn_args {
    const void* qkv; int64_t ld_qkv; int32_t q_col, k_col, v_col;
    const int32_t* seqlens; int32_t B, L, heads;
    void* out; int64_t ldo; int32_t out_col_offset;
    void* const* out_peers; int32_t world, rows_per_rank;
    float score_bound_log2;
    int32_t schedule;            /* VCB_ATTN_SCHED_* ; 0 = auto */
} vcb_attn_args;
int vcb_attention_fwd_ex(const vcb_attn_args* args, void* stream);
/* debug aid (environment VCB_ATTN4_TIMELINE=1): per-CTA globaltimer stamps [grid][66] (start, end of every segment) of the most
 * recent persistent attention launch; synchronises the device; returns the grid size or -1 */
int vcb_debug_attn4_timeline(unsigned long long* out, int32_t capacity);

/* ---- AdaLN modulated LayerNorm (layers.py:163-164,191,195,234,257):
 *      y = bf16( bf16(1 + scale[b]) * LayerNorm(x) + shift[b] ), eps 1e-6, no affine.
 *      Every vcb_ln_modulate* entry point needs hidden % 256 == 0 and hidden <= 6144 (the modulation vectors of a block are
 *      staged in 8 * hidden bytes of shared memory).
 *      Logical row r = (b, i) with b = r / rows_per_batch lives at physical row b * batch_rows + i of x and y
 *      (batch_rows = 0 means rows_per_batch, i.e. a plain [rows, hidden] matrix). */
int vcb_ln_modulate(const void* x, int64_t ldx, void* y, int64_t ldy, const void* shift, const void* scale,
                    int64_t mod_stride, int32_t rows, int32_t hidden, int32_t rows_per_batch, int32_t batch_rows,
                    void* stream);

/* Two row ranges of the same [*, hidden] buffers with their own modulation vectors in ONE launch (the img and txt streams of
 * a DoubleStreamBlock): ldx / ldy / mod_stride / hidden / batch_rows (> 0) are shared.  a1 may be NULL: one problem. */
typedef struct vcb_ln_args { const void* x; void* y; const void* shift; const void* scale; int32_t rows, rows_per_batch; } vcb_ln_args;
int vcb_ln_modulate_grouped(const vcb_ln_args* a0, const vcb_ln_args* a1, int64_t ldx, int64_t ldy, int64_t mod_stride,
                            int32_t hidden, int32_t batch_rows, void* stream);

/* Statistics supplied by the producer: stats0 / stats1 [rows of the problem][n_slots] float2 as written by the row_stats member of
 * the VCB_EPI_GATE_RES GEMM that produced x (positioned at the problem's first row); the kernel adds a row's n_slots pairs in a
 * fixed order and streams the row once.  One or two problems per launch (a1 / stats1 may be NULL). */
int vcb_ln_modulate_stats(const vcb_ln_args* a0, const vcb_ln_args* a1, const void* stats0, const void* stats1, int32_t n_slots,
                          int64_t ldx, int64_t ldy, int64_t mod_stride, int32_t hidden, int32_t batch_rows, void* stream);

/* FP8 form (opt-in fp8 projections): same LayerNorm + modulation, but the output row is e4m3 bytes (y8 [*, ld8], bytes) with one
 * fp32 scale per row, row_scale[physical row] = max|y| / 448 -- the a_scale of the fp8 GEMM that consumes it.  One or two
 * problems per launch (a1 may be NULL); vcb_ln_args.y is then the e4m3 destination of that problem. */
int vcb_ln_modulate_fp8(const vcb_ln_args* a0, const vcb_ln_args* a1, float* row_scale0, float* row_scale1, int64_t ldx, int64_t ld8,
                        int64_t mod_stride, int32_t hidden, int32_t batch_rows, void* stream);
/* the same with the row statistics supplied by the producing GEMM (see vcb_ln_modulate_stats) */
int vcb_ln_modulate_fp8_stats(const vcb_ln_args* a0, const vcb_ln_args* a1, float* row_scale0, float* row_scale1, const void* stats0,
                              const void* stats1, int32_t n_slots, int64_t ldx, int64_t ld8, int64_t mod_stride, int32_t hidden,
                              int32_t batch_rows, void* stream);

/* Row-wise e4m3 quantisation of a bf16 matrix x [rows, K] (row stride ldx elements; K % 8 == 0, K <= 15360): y8 [rows, K] e4m3
 * bytes (row stride ld8 bytes) and row_scale[row] = max(max|x|, 1e-12) / 448, so that x ~= y8 * row_scale.  Feeds the fp8 form of
 * the Linears whose input is NOT a LayerNorm output (fp8 level 2: attn.proj, mlp.2, linear2 -- layers.py:190-195, 244). */
int vcb_quantize_rows_e4m3(const void* x, int64_t ldx, void* y8, int64_t ld8, float* row_scale, int64_t rows, int32_t K,
                           void* stream);

/* ---- text encoders (SURVEY 8f-4): the reference wraps HF T5EncoderModel("google/t5-v1_1-xxl") and CLIPTextModel(
 * "openai/clip-vit-large-patch14") in models/modules/conditioner.py:5-37 (bf16, models/util.py:425-431) and calls them with
 * attention_mask=None.  Their Linears run through vcb_gemm_bf16; these entry points are everything else.  All tensors bf16. -------- */
/* out[t, :] = table[ids[t], :] (+ pos_table[t % L, :] when pos_table != NULL: CLIP's token + position embedding); ids int64 */
int vcb_embedding_bf16(const void* table, int64_t vocab, int32_t dim, const int64_t* ids, const void* pos_table, int32_t L,
                       void* out, int64_t ldo, int64_t n_tokens, void* stream);
/* T5LayerNorm: y = weight * bf16(x * rsqrt(mean(x^2) + eps)), fp32 statistics, no mean subtraction, no bias */
int vcb_rmsnorm_weight(const void* x, int64_t ldx, const void* weight, void* y, int64_t ldy, int64_t rows, int32_t dim, float eps,
                       void* stream);
/* nn.LayerNorm with affine parameters (CLIP): y = bf16((x - mean) * rstd * weight + bias), fp32 statistics */
int vcb_layernorm_affine(const void* x, int64_t ldx, const void* weight, const void* bias, void* y, int64_t ldy, int64_t rows,
                         int32_t dim, float eps, void* stream);
/* T5DenseGatedActDense: out[:, j] = gelu_new(ab[:, j]) * ab[:, dff + j] (wi_0 and wi_1 computed by ONE GEMM of width 2 * dff) */
int vcb_gated_gelu(const void* ab, int64_t ld, void* out, int64_t ldo, int64_t rows, int32_t dff, void* stream);
/* CLIP's quick_gelu: y = x * sigmoid(1.702 x) */
int vcb_quick_gelu(const void* x, void* y, int64_t n, void* stream);
/* attention of the two text encoders: head_dim 64, L <= 512, row (b * L + i) of q / k / v with head h at column h * 64 (row stride
 * ld: the three may point into one fused [B * L, 3 * heads * 64] buffer); scores = bf16(q k^T) (* scale), + bias[h, i, j] (T5's
 * relative position bias, may be NULL), causal mask (CLIP), fp32 softmax, bf16 probabilities -- the HF modules' rounding points */
typedef struct vcb_attn_small_args {
    const void* q; const void* k; const void* v; int64_t ld;
    const void* bias;            /* [heads, L, L] bf16 or NULL */
    void* out; int64_t ldo;      /* [B * L, heads * 64] */
    int32_t B, L, heads, head_dim, causal;
    float scale;                 /* 0 or 1 = no scaling (T5); CLIP: head_dim^-0.5 */
} vcb_attn_small_args;
int vcb_attention_small(const vcb_attn_small_args* a, void* stream);

/* ---- small helpers --------------------------------------------------------------------------------------- */
/* layers.py:28-49; t_scaled = time_factor * t already in the reference's dtype; freqs[128] fp32; out [n,256] bf16 */
int vcb_timestep_embedding(const float* t_scaled, const float* freqs, void* out, int32_t n, void* stream);
int vcb_silu(const void* x, void* y, int64_t n, void* stream);
/* out[r] = bf16(bf16(a[r] + b[r % b_rows]) + c[r % c_rows]); b, c may be NULL   (model.py:102-107) */
int vcb_add3(const void* a, const void* b, int32_t b_rows, const void* c, int32_t c_rows, void* out,
             int32_t rows, int32_t hidden, void* stream);
/* layers.py:11-25 + math.py:102-109: ids [rows,3] fp32 -> (cos,sin) float2, PAIR-MAJOR [64][rows] */
int vcb_rope_table(const float* ids, void* out, int32_t rows, int32_t d0, int32_t d1, int32_t d2, double theta,
                   void* stream);
/* torchdiffeq euler step as used by transport/integrators.py:119 (bf16 state, dt rounded to bf16, v negated);
 * model_in may be NULL, else x_new is also written into its first C columns. */
int vcb_euler_update(const void* x, const void* v, float dt_bf16, void* x_new, void* model_in, int64_t ld_in,
                     int64_t rows, int32_t C, void* stream);
/* One stage update of torchdiffeq's fixed-grid solvers (torchdiffeq/_impl/fixed_grid.py, rk_common.py; unpinned) as
 * transport/integrators.py:119 calls them, on one interval [t0, t1] of a bf16 state.  dt = the fp32 value of t1 - t0;
 * v = host array of the n_v = stage + 1 model outputs v_1..v_{stage+1} of this interval, each [rows, C] bf16, where the
 * solver's k_i = -v_i (transport.py:384).  y_out [rows, C] receives the result; model_in (may be NULL, leading dimension
 * ld_in >= C) also receives it in columns [0, C), the rest of each row (`cond`) is left as it is.  The result equals, bit for
 * bit, the eager torch expression with y0, k_i bf16 tensors, dt a 0-dim fp32 tensor and _one_third = 1/3 a Python float:
 *   VCB_ODE_EULER     stage 0:  y0 + dt * k1
 *   VCB_ODE_MIDPOINT  stage 0:  y0 + k1 * half_dt            (half_dt = 0.5 * dt; the state k2 is evaluated at)
 *                     stage 1:  y0 + dt * k2                 (the next grid point)
 *   VCB_ODE_RK4       stage 0:  y0 + dt * k1 * _one_third    (the 3/8 rule, rk4_alt_step_func: the state of k2)
 *                     stage 1:  y0 + dt * (k2 - k1 * _one_third)                   (the state of k3)
 *                     stage 2:  y0 + dt * (k1 - k2 + k3)                           (the state of k4)
 *                     stage 3:  y0 + (k1 + 3 * (k2 + k3) + k4) * dt * 0.125       (the next grid point)
 * 16-byte accesses when C and ld_in are multiples of 8 and every pointer is 16-byte aligned; any layout works. */
#define VCB_ODE_EULER 0
#define VCB_ODE_MIDPOINT 1
#define VCB_ODE_RK4 2
int vcb_ode_stage(int32_t method, int32_t stage, const void* y0, const void* const* v, int32_t n_v, float dt,
                  void* y_out, void* model_in, int64_t ld_in, int64_t rows, int32_t C, void* stream);
int vcb_copy_cols(const void* src, int64_t lds, void* dst, int64_t ldd, int32_t col0, int64_t rows, int32_t C,
                  void* stream);


/* ---- FLUX-DiT engine: the whole Flux.forward (models/model.py:85-124) and the Euler loop around it -----------
 * Weights are the reference's tensors in one of two forms, chosen per Linear (lora.py:92-98): LoRA merged (rank 0:
 * w = W + s*B*A) or unmerged (rank > 0: w = W, lora_a = A [rank, in], lora_b = B [out, rank], lora_scale = s; every call then
 * runs the down-projection T = bf16(s * x A^T) and the main GEMM with the LoRA k-tail, vcb_gemm_args.lora_*).  Either way
 * b = b + s*b_B; bf16 weights [out, in], fp32 biases.  The engine keeps pointers only; the caller owns weights and workspace. */
/* w8 / w8_scale (optional): the same merged weight quantised to e4m3 with one fp32 scale per output channel (w ~= w8 * scale),
 * used by the opt-in fp8 projections (vcb_flux_set_fp8): level 1 needs it on the LayerNorm-fed Linears (qkv, mlp.0, linear1), level 2
 * also on attn.proj, mlp.2 and linear2; NULL = bf16 only. */
/* lora_a / lora_b / rank / lora_scale: the unmerged LoRA form (rank % 8 == 0; rank 0 or lora_scale 0 = no update); bf16 only, so
 * an engine holding an unmerged Linear refuses vcb_flux_set_fp8 and vcb_flux_sp_attach. */
typedef struct vcb_linear_w {
    const void* w; const float* b; const void* w8; const float* w8_scale;
    const void* lora_a; const void* lora_b; int32_t rank; float lora_scale;
} vcb_linear_w;

typedef struct vcb_stream_w {           /* one stream of a DoubleStreamBlock (layers.py:129-156) */
    vcb_linear_w mod, qkv, proj, mlp0, mlp2;
    const void* q_scale; const void* k_scale;      /* [128] bf16 */
} vcb_stream_w;
/* attn_score_bound: 0, or an upper bound (log2 units) of the block's scaled attention scores derived from its QK-norm scales
 * = max|q_scale| * max|k_scale| * sqrt(128) * log2(e) * (1 + margin); see vcb_attn_args.score_bound_log2 */
typedef struct vcb_double_w { vcb_stream_w img, txt; float attn_score_bound; } vcb_double_w;
typedef struct vcb_single_w {           /* SingleStreamBlock (layers.py:199-230) */
    vcb_linear_w mod, linear1, linear2;
    const void* q_scale; const void* k_scale;
    float attn_score_bound;
} vcb_single_w;

typedef struct vcb_flux_config {        /* FluxParams (models/model.py:18-32) */
    int32_t in_channels, out_channels, vec_in_dim, context_in_dim, hidden, mlp_hidden, heads;
    int32_t depth, depth_single, axes_dim[3], guidance_embed;
    double theta;
} vcb_flux_config;

typedef struct vcb_flux_weights {
    vcb_linear_w img_in, txt_in, time_in0, time_in1, vector_in0, vector_in1, guidance_in0, guidance_in1;
    vcb_linear_w final_mod, final_linear;
    const vcb_double_w* dbl;            /* host array [depth] */
    const vcb_single_w* sgl;            /* host array [depth_single] */
} vcb_flux_weights;

typedef struct vcb_flux vcb_flux;       /* opaque */

int  vcb_flux_create(const vcb_flux_config* cfg, const vcb_flux_weights* w, vcb_flux** out);
void vcb_flux_destroy(vcb_flux* f);
/* enable (default) / disable the per-block attn_score_bound: disabled, every block runs the exact online-max softmax -- what a
 * checkpoint whose QK-norm scales leave the safe range gets anyway; used to measure that path on any weights */
int  vcb_flux_use_score_bounds(vcb_flux* f, int32_t enable);
/* opt-in FP8 (e4m3) projections: the Linears fed by an AdaLN LayerNorm (double blocks: img/txt qkv and mlp.0; single blocks:
 * linear1 -- 58 % of the step's GEMM FLOPs) run on e4m3 wgmma with per-row activation scales (written by the
 * LayerNorm kernel) and per-output-channel weight scales; everything else stays bf16.  Needs the w8 / w8_scale members of those
 * weights.  level 2 (VCB_FP8_ALL_LINEARS) adds the gated-residual Linears (attn.proj, mlp.2, linear2 -- all of the blocks' GEMM
 * FLOPs): their bf16 inputs (attention output, GELU output) are quantised row-wise by vcb_quantize_rows_e4m3 first.
 * NOT the reference's numerics: a separate tolerance contract applies per level (DESIGN.md, tests/test_fp8_gpu.py). */
#define VCB_FP8_OFF 0
#define VCB_FP8_LN_FED 1
#define VCB_FP8_ALL_LINEARS 2
int  vcb_flux_set_fp8(vcb_flux* f, int32_t level);
/* bytes of device workspace for B samples of Li image + Lt text tokens and n_evals model evaluations (with unmerged LoRA
 * Linears: + the down-projection buffer T [max(B * (Li + Lt), n_evals * B), largest rank] bf16; with the first-block cache on:
 * + its buffers, vcb_flux_set_first_block_cache) */
int64_t vcb_flux_workspace_bytes(const vcb_flux* f, int32_t B, int32_t Li, int32_t Lt, int32_t n_evals);
/* Step-invariant work, once per image (SURVEY.md 2.2: txt_in, RoPE table, and the AdaLN modulation vectors of
 * all n_evals steps as one batched GEMM per block).  t_scaled: [n_evals * B] fp32 = 1000 * flux_time (row e*B+b);
 * g_scaled: [B] fp32 = float(bf16(1000 * guidance)) or NULL; freqs: [128] fp32 (layers.py:39); txt [B,Lt,ctx] bf16;
 * y [B, vec_in] bf16; ids [B, Lt+Li, 3] fp32 (txt ids first); seqlens [B] int32 valid tokens of the joint
 * sequence (Lt + valid img tokens) or NULL. */
int vcb_flux_prepare(vcb_flux* f, void* workspace, int64_t workspace_bytes, int32_t B, int32_t Li, int32_t Lt,
                     int32_t n_evals, const void* txt, const void* y, const float* ids, const float* t_scaled,
                     const float* g_scaled, const float* freqs, const int32_t* seqlens, void* stream);
/* One model evaluation (Flux.forward) with the tables of evaluation `eval_idx`:
 * img [B*Li, in_channels] bf16 (latent || cond) -> out [B*Li, out_channels] bf16. */
int vcb_flux_forward(vcb_flux* f, int32_t eval_idx, const void* img, int64_t ld_img, void* out, int64_t ld_out,
                     void* stream);
/* Opt-in first-block cache (FBCache; off by default; NOT the reference's numerics).  threshold > 0 switches it on, 0 off.  Per
 * vcb_flux_prepare, evaluation k runs img_in and double block 0 as usual; with x0 / x1 the img rows of x before / after that
 * block, r_k = bf16(x1 - x0) and diff_k = sum|r_k - r_ref| / sum|r_ref| (fp32, fixed summation order, valid img rows of every
 * sample: right padding excluded through seqlens; one decision per batch).  k > 0 and diff_k < threshold: the img rows become
 * bf16(x1 + R) and go straight to the final layer.  Otherwise blocks 1.. run, r_ref = r_k and R = x_final - x1 (fp32) are kept.
 * The first evaluation after every prepare is computed.  While on, the final LayerNorm computes its own row statistics (also on
 * computed evaluations), and vcb_flux_forward reads the decision on the host: it synchronises `stream` once per call and cannot be
 * captured in a CUDA graph.  The workspace grows by B * Li * hidden * 8 bytes (x0 / r_ref bf16 pair + R fp32).  Refused in
 * sequence-parallel mode (and vcb_flux_sp_attach refuses while it is on); needs depth >= 1. */
int vcb_flux_set_first_block_cache(vcb_flux* f, float threshold);
/* evaluations computed / skipped since the last vcb_flux_prepare, and diff of the latest one (+inf for the first evaluation after
 * prepare, which has nothing to compare with; NaN before any) */
int vcb_flux_cache_stats(const vcb_flux* f, int32_t* computed, int32_t* skipped, float* last_diff);

/* ---- single-image sequence parallelism over NVLink peer memory (SURVEY.md 8f-2: the reference has no multi-GPU
 * inference; the join point is the attention call, layers.py:177-187 / 236-241) -----------------------------------
 * W ranks (one process per GPU) each hold a full weight copy and 1/W of the txt rows and 1/W of the img rows of ONE
 * sample.  Everything except attention is row-local.  For attention, rank s owns heads [s*heads/W, (s+1)*heads/W):
 * the QKV GEMM epilogue scatters q/k/v by head into the owners' qkv buffers and the attention epilogue scatters its
 * output rows back to the row owners' `cat` buffers, both as plain stores to cudaIpc-mapped peer memory; a flag
 * barrier (system-scope release/acquire) separates the phases.  No NCCL call on the per-step path.
 *
 * vcb_peer_alloc / vcb_peer_open: zero-filled device memory that other processes on the node can map.  handle = 64 opaque bytes to
 * pass to the peers (any host channel); vcb_peer_open maps a peer's allocation into this process (enables P2P). */
int vcb_peer_alloc(int64_t bytes, void** ptr, void* handle64);
int vcb_peer_open(const void* handle64, void** ptr);
int vcb_peer_close(void* ptr);
int vcb_peer_free(void* ptr);
/* All-ranks barrier on `stream`: publishes epoch to every peer's flag word [rank] and waits until every peer has
 * published >= epoch to ours.  flags[r] = rank r's int32[VCB_SP_MAX] flag array (peer-mapped for r != rank), zeroed
 * before first use; epochs must increase by one per call, identically on all ranks.  err (device int32, local) is set
 * to the epoch if a peer does not arrive within timeout_ms (the kernel then exits instead of hanging the GPU). */
int vcb_sp_barrier(int32_t* const* flags, int32_t world, int32_t rank, int32_t epoch, int32_t* err, int32_t timeout_ms,
                   void* stream);
/* Shared buffers a rank must vcb_peer_alloc for Li_local + Lt_local rows: qkv [(W*L_local), 3*hidden/W] and
 * cat [L_local, hidden + mlp_hidden], bf16. */
int vcb_flux_sp_shared_bytes(const vcb_flux* f, int32_t Li_local, int32_t Lt_local, int64_t* qkv_bytes, int64_t* cat_bytes);
/* Switch the engine to sequence-parallel mode (world == 1 switches back).  qkv/cat/flags: arrays [world] of the ranks'
 * buffers as mapped in THIS process (entry [rank] is the local allocation).  vcb_flux_prepare / vcb_flux_forward then
 * take LOCAL sizes: B == 1, Li = Li_local, Lt = Lt_local, ids / txt / img / out rows of this rank only, seqlens NULL. */
int vcb_flux_sp_attach(vcb_flux* f, int32_t world, int32_t rank, void* const* qkv, void* const* cat, int32_t* const* flags,
                       int32_t* err, int32_t timeout_ms);

/* ---- VAE decoder (models/modules/autoencoder.py:183-259, 307-309; the pipeline's AutoencoderKL.decode, visualcloze.py:430)
 * NHWC bf16 activations; 3x3 convs as implicit wgmma GEMMs, GroupNorm(32)+swish, nearest-2x upsampling and the
 * single-head mid-block attention as HBM-bound kernels.  Conv weights are [cout, 3, 3, cin_padded] bf16 (tap-major,
 * channels last, cin padded to a multiple of 64, cout of conv_out padded to 8), 1x1 convs [cout, cin]; biases and
 * GroupNorm affine parameters fp32. */
typedef struct vcb_conv_w { const void* w; const float* b; int32_t cin, cout; } vcb_conv_w;
typedef struct vcb_gn_w { const float* gamma; const float* beta; } vcb_gn_w;
typedef struct vcb_resblock_w {            /* ResnetBlock, autoencoder.py:55-82 */
    vcb_gn_w norm1; vcb_conv_w conv1; vcb_gn_w norm2; vcb_conv_w conv2;
    vcb_conv_w shortcut;                   /* 1x1 nin_shortcut; w == NULL when cin == cout */
} vcb_resblock_w;
typedef struct vcb_vae_config {
    int32_t ch, out_ch, z_channels, num_res_blocks, n_levels;
    int32_t ch_mult[8];
    float scale_factor, shift_factor;
} vcb_vae_config;
typedef struct vcb_vae_weights {
    vcb_conv_w conv_in;
    vcb_resblock_w mid1, mid2;
    vcb_gn_w attn_norm;
    vcb_conv_w attn_q, attn_k, attn_v, attn_proj;          /* 1x1 convs == linear layers over channels */
    const vcb_resblock_w* up_blocks;       /* host array, execution order: level n-1 .. 0, num_res_blocks+1 each */
    const vcb_conv_w* upsample;            /* host array, execution order: one per level except level 0 */
    vcb_gn_w norm_out;
    vcb_conv_w conv_out;
} vcb_vae_weights;
typedef struct vcb_vae vcb_vae;

int  vcb_vae_create(const vcb_vae_config* cfg, const vcb_vae_weights* w, vcb_vae** out);
void vcb_vae_destroy(vcb_vae* v);
/* workspace for n latents of h x w packed tokens (latent 2h x 2w, image 16h x 16w for the 4-level FLUX VAE) */
int64_t vcb_vae_workspace_bytes(const vcb_vae* v, int32_t n, int32_t h, int32_t w);
/* tokens [n, h*w, 4*z_channels] bf16 -> raw [n, out_ch, H, W] fp32 (decoder output, may be NULL) and/or
 * img [n, out_ch, H, W] uint8 = to_pil(clamp((x + 1) / 2, 0, 1)) (may be NULL) */
int vcb_vae_decode(vcb_vae* v, void* workspace, int64_t workspace_bytes, const void* tokens, int32_t n, int32_t h,
                   int32_t w, float* raw, uint8_t* img, void* stream);

/* ---- VAE encoder (models/modules/autoencoder.py:109-180, 262-275, 302-305; the pipeline's ae.encode(...).latent_dist.sample(),
 * visualcloze.py:377-388) -- "next" row (f)-1 of SURVEY.md section 8: same kernels as the decoder, stride-2 convs through
 * TMA element strides.  Weights as for the decoder (conv_in cin padded to 64). */
typedef struct vcb_vae_enc_weights {
    vcb_conv_w conv_in;
    const vcb_resblock_w* down_blocks;     /* host array, execution order: level 0 .. n-1, num_res_blocks each */
    const vcb_conv_w* downsample;          /* host array: one stride-2 conv per level except the last */
    vcb_resblock_w mid1, mid2;
    vcb_gn_w attn_norm;
    vcb_conv_w attn_q, attn_k, attn_v, attn_proj;
    vcb_gn_w norm_out;
    vcb_conv_w conv_out;                   /* -> 2 * z_channels (mean | logvar) */
} vcb_vae_enc_weights;
typedef struct vcb_vae_enc vcb_vae_enc;
int  vcb_vae_enc_create(const vcb_vae_config* cfg, const vcb_vae_enc_weights* w, vcb_vae_enc** out);
void vcb_vae_enc_destroy(vcb_vae_enc* e);
int64_t vcb_vae_enc_workspace_bytes(const vcb_vae_enc* e, int32_t n, int32_t H, int32_t W);
/* image [n, 3, H, W] fp32 in [-1, 1] (H, W multiples of 16) -> packed condition tokens [n, (H/16)(W/16), 4*z] bf16 =
 * patchify((sample - shift) * scale), sample = mean + exp(0.5 logvar) * noise (noise [n, z, H/8, W/8] fp32; NULL = mode);
 * moments (optional): raw encoder output [n, 2z, H/8, W/8] fp32. */
int vcb_vae_encode(vcb_vae_enc* e, void* workspace, int64_t workspace_bytes, const float* image, int32_t n, int32_t H,
                   int32_t W, const float* noise, void* tokens, float* moments, void* stream);

/* ---- test hook: one 128x128x(16*ksteps) wgmma tile with caller-chosen descriptor fields -------------------
 * Used by tests/ to pin the shared-memory / register operand layouts the kernels rely on.  a: [128, K] bf16 (K-major),
 * b: B operand, either [128(N), K] K-major (b_mn_major=0) or [K, 128(N)] N-contiguous (b_mn_major=1);
 * a_from_regs: feed A from registers (the accumulator's row layout) instead of smem.  out: [128,128] fp32. */
int vcb_debug_umma_probe(const void* a, const void* b, float* out, int32_t ksteps, int32_t b_mn_major,
                         int32_t a_from_regs, uint32_t b_lbo, uint32_t b_sbo, uint32_t b_kstep_bytes, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* VCB200_H_ */
