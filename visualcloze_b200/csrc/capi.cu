// capi.cu -- extern "C" boundary of libvcb200.so (see include/vcb200.h) and the host-side launch code.
#include <atomic>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <mutex>

#include "../../include/vcb200.h"
#include "attn_sm90.cuh"
#include "elementwise.cuh"
#include "gemm_sm90.cuh"
#include "host_util.cuh"
#include "probe.cuh"
#include "sp_sm90.cuh"

using namespace vcb;

// ------------------------------------------------------------------------------------------------
// GEMM dispatch
// ------------------------------------------------------------------------------------------------
namespace {

struct Problem { CUtensorMap ta, tb, tt, tl; GemmParams p; };      // tt / tl: LoRA k-tail maps (T, lora_b); copies of ta / tb without one

// stream-K scratch: one slot of 128 x 256 fp32 per CTA and one flag per CTA, per stream (launches on one stream are
// ordered, so a single scratch per stream is enough); allocated on first use (call once before CUDA-graph capture)
struct SkScratch { float* ws = nullptr; int* flags = nullptr; int epoch = 0; };
inline SkScratch* sk_scratch(cudaStream_t st) {
    static std::mutex mu;
    static std::map<cudaStream_t, SkScratch> pool;
    std::lock_guard<std::mutex> lk(mu);
    SkScratch& s = pool[st];
    if (!s.ws) {
        const size_t n = 160;                                  // >= number of SMs
        if (cudaMalloc(&s.ws, n * 128 * 256 * sizeof(float)) != cudaSuccess) return nullptr;
        if (cudaMalloc(&s.flags, n * sizeof(int)) != cudaSuccess) return nullptr;
        cudaMemset(s.flags, 0, n * sizeof(int));
    }
    return &s;
}
// Stream-K policy.  VCB_STREAMK unset = auto, 0 = never, 1 = whenever feasible and the estimated saving exceeds 20 us.
// Auto enables the tail split only when the idle part of the last wave is a large share of the WHOLE launch (>= 20 %) --
// the few-wave GEMMs of the sequence-parallel mode; with many waves the partial exchange costs more than the idle tail.
inline int streamk_mode() {
    static const int m = [] { const char* e = getenv("VCB_STREAMK"); return e ? (atoi(e) ? 1 : 0) : -1; }();
    return m;
}
constexpr float kSkOverheadUs = 30.f;      // estimate: partial dump + fold of a split tile, waiting for the partners (tools/bench_sk.py measures it)
// time of one output tile (us) for a configuration with the full-wave rate `rate` (TFLOP/s over all SMs)
inline float tile_time_us(int bn, int K, float rate) { return 2.f * 128.f * bn * (float)K * (float)num_sms() / (rate * 1e6f); }
inline bool streamk_feasible(long tiles, int slots) {
    // also with fewer tiles than CTA slots (one partial "wave"): every slot then gets an equal K range of the few tiles
    const long rem = tiles % slots;
    return rem != 0 && rem * (kSkMaxParts - 1) >= slots && num_sms() <= 160;
}
inline bool streamk_wanted(long tiles, int slots, float tile_us) {
    const int mode = streamk_mode();
    if (mode == 0 || !streamk_feasible(tiles, slots)) return false;
    const long waves = (tiles + slots - 1) / slots;
    const float idle = 1.0f - (float)(tiles % slots) / slots;
    if (idle * tile_us <= (mode < 0 ? kSkOverheadUs : 20.f)) return false;   // the split must save more than it costs
    return mode == 1 || idle / waves >= 0.2f;
}

template <int BN, int CG, int EPI, bool SP = false, bool FP8 = false>
int launch_gemm_inst(const Problem& g0, const Problem& g1, float rate, cudaStream_t st) {
    const CUtensorMap& ta = g0.ta; const CUtensorMap& tb = g0.tb; const GemmParams& p = g0.p;
    using Cfg = GemmCfg<BN, CG>;
    auto kern = gemm_wgmma_kernel<BN, CG, EPI, A_MATRIX, SP, FP8>;
    constexpr int kSmem = Cfg::kSmemBytes;
    static std::once_flag once;
    static cudaError_t attr_err = cudaSuccess;
    std::call_once(once, [&] {
        attr_err = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmem);
    });
    if (attr_err != cudaSuccess) return set_error("cudaFuncSetAttribute(gemm): %s", cudaGetErrorString(attr_err));
    const int tile_m = kBlockM * CG;
    int tiles = p.batch * ((p.rows_per_batch + tile_m - 1) / tile_m) * ((p.N + BN - 1) / BN);
    if (g1.p.batch > 0) tiles += g1.p.batch * ((g1.p.rows_per_batch + tile_m - 1) / tile_m) * ((p.N + BN - 1) / BN);
    int clusters = num_sms() / CG;
    // stream-K tail: the tiles of the partial last wave are cut along K into one equal range per CTA (pair)
    StreamKParams skp{nullptr, nullptr, 0, 0};
    const bool sk = streamk_wanted(tiles, clusters, tile_time_us(BN, p.K + p.lora_rank, rate) * (FP8 ? 0.5f : 1.0f));
    if (tiles < clusters && !sk) clusters = tiles;
    if (sk) {
        SkScratch* sc = sk_scratch(st);
        if (!sc) return set_error("gemm: stream-K scratch allocation failed");
        skp.ws = sc->ws; skp.flags = sc->flags; skp.epoch = ++sc->epoch; skp.enabled = 1;
    }
    cudaError_t e = launch_pdl(kern, dim3(clusters * CG), dim3(kGemmThreads), (size_t)kSmem, st, CG, ta, tb, p, g1.ta, g1.tb, g1.p, skp,
                               g0.tt, g0.tl, g1.tt, g1.tl);
    if (e != cudaSuccess) return set_error("gemm launch (BN=%d CG=%d EPI=%d): %s", BN, CG, EPI, cudaGetErrorString(e));
    count_launch();
    return 0;
}

// fp8 operands: the LayerNorm-fed projections of the FLUX blocks (qkv, mlp-up, linear1), plain bias GEMMs and -- level 2, A
// quantised by vcb_quantize_rows_e4m3 -- the gated-residual projections (proj, mlp-down, linear2)
template <int BN, int CG>
int launch_gemm_epi_fp8(int epi, const Problem& g0, const Problem& g1, float rate, cudaStream_t st) {
    if (epi == EPI_BIAS) return launch_gemm_inst<BN, CG, EPI_BIAS, false, true>(g0, g1, rate, st);
    if (epi == EPI_BIAS_GELU) return launch_gemm_inst<BN, CG, EPI_BIAS_GELU, false, true>(g0, g1, rate, st);
    if (epi == EPI_GATE_RES) return launch_gemm_inst<BN, CG, EPI_GATE_RES, false, true>(g0, g1, rate, st);
    if constexpr (BN % 128 == 0) {
        if (epi == EPI_QKV) return launch_gemm_inst<BN, CG, EPI_QKV, false, true>(g0, g1, rate, st);
        if (epi == EPI_LINEAR1) return launch_gemm_inst<BN, CG, EPI_LINEAR1, false, true>(g0, g1, rate, st);
    }
    return set_error("gemm (fp8): epilogue %d not available for block_n %d", epi, BN);
}

template <int BN, int CG>
int launch_gemm_epi(int epi, const Problem& g0, const Problem& g1, float rate, cudaStream_t st) {
    switch (epi) {
        case EPI_BIAS: return launch_gemm_inst<BN, CG, EPI_BIAS>(g0, g1, rate, st);
        case EPI_BIAS_GELU: return launch_gemm_inst<BN, CG, EPI_BIAS_GELU>(g0, g1, rate, st);
        case EPI_GATE_RES: return launch_gemm_inst<BN, CG, EPI_GATE_RES>(g0, g1, rate, st);
        case EPI_BIAS_F32: return launch_gemm_inst<BN, CG, EPI_BIAS_F32>(g0, g1, rate, st);
        default: break;
    }
    if constexpr (BN % 128 == 0) {
        const bool sp = g0.p.sp_world > 1;        // sequence-parallel: stores through the owners' peer-mapped buffers
        if (epi == EPI_QKV) return sp ? launch_gemm_inst<BN, CG, EPI_QKV, true>(g0, g1, rate, st) : launch_gemm_inst<BN, CG, EPI_QKV>(g0, g1, rate, st);
        if (epi == EPI_LINEAR1) return sp ? launch_gemm_inst<BN, CG, EPI_LINEAR1, true>(g0, g1, rate, st) : launch_gemm_inst<BN, CG, EPI_LINEAR1>(g0, g1, rate, st);
    }
    return set_error("gemm: epilogue %d not available for block_n %d", epi, BN);
}

int forced_cta_group() {
    static int v = [] {
        const char* e = getenv("VCB_GEMM_CTA_GROUP");
        return e ? atoi(e) : 0;
    }();
    return v;
}

// Tile selection.  Cost of a configuration = (tiles per CTA slot, rounded up) x (tile width) / (full-wave rate of that
// configuration, TFLOP/s over all SMs).  The rates are relative weights, not measurements: wider tiles re-read less of A per
// FLOP, cta_group 2 pairs two SMs on a 256 x BLOCK_N tile and fetches each B tile from L2 once for both; narrow tiles win when
// they remove a partial wave.  tools/bench_kernels.py measures the configurations.
struct TileCfg { int cg, bn; float rate; };
constexpr TileCfg kTileCfgs[] = {{1, 256, 600.f}, {2, 256, 600.f}, {1, 192, 560.f}, {2, 192, 560.f},
                                 {1, 128, 500.f}, {2, 128, 500.f}};

void pick_tile(int batch, int rows, int N, int K, bool head_structured, int want_cg, int want_bn, int* cg_out, int* bn_out,
               float* rate_out) {
    float best_cost = -1.f, best_rate = 600.f;
    int best_cg = 1, best_bn = 256;
    for (const TileCfg& c : kTileCfgs) {
        if (want_cg && c.cg != want_cg) continue;
        if (want_bn && c.bn != want_bn) continue;
        if (head_structured && c.bn % 128) continue;
        const int slots = num_sms() / c.cg;
        const long mt = (long)batch * ((rows + kBlockM * c.cg - 1) / (kBlockM * c.cg));
        const long tiles = mt * ((N + c.bn - 1) / c.bn);
        const long waves = (tiles + slots - 1) / slots;
        const float tile_us = tile_time_us(c.bn, K, c.rate);
        // with the stream-K tail the last wave costs its filled fraction (+ the partial exchange) instead of a whole wave
        const float cost = streamk_wanted(tiles, slots, tile_us) ? (float)tiles / slots * tile_us + kSkOverheadUs : (float)waves * tile_us;
        if (best_cost < 0.f || cost < best_cost) { best_cost = cost; best_cg = c.cg; best_bn = c.bn; best_rate = c.rate; }
    }
    if (best_cost < 0.f) { best_cg = want_cg ? want_cg : 1; best_bn = want_bn ? want_bn : 256; }   // e.g. block_n 64
    *cg_out = best_cg;
    *bn_out = best_bn;
    *rate_out = best_rate;
}

}  // namespace

namespace {

// validate one problem
int check_gemm_args(const vcb_gemm_args* a) {
    if (!a) return set_error("gemm: null args");
    if (a->M <= 0 || a->N <= 0 || a->K <= 0) return set_error("gemm: bad shape %d %d %d", a->M, a->N, a->K);
    if (a->lda % 8 || a->ldw % 8 || a->ldo % 8 || a->out_col_offset % 8)
        return set_error("gemm: leading dims and column offsets must be multiples of 8 (16-byte rows)");
    // N need not be a multiple of 8 when the output row has room for the rounded-up width: the extra columns receive the
    // epilogue of TMA-zero-filled weight rows.  K is arbitrary (the TMA unit zero-fills the k tail of both operands).
    if (a->N % 8 && (a->epilogue != VCB_EPI_BIAS && a->epilogue != VCB_EPI_BIAS_F32))
        return set_error("gemm: N must be a multiple of 8 for this epilogue");
    if (a->N % 8 && a->out_col_offset + (a->N + 7) / 8 * 8 > a->ldo)
        return set_error("gemm: N %% 8 != 0 needs ldo >= out_col_offset + round_up(N, 8)");
    if (!a->A || !a->W || !a->out) return set_error("gemm: null operand");
    const bool head = a->epilogue == VCB_EPI_QKV || a->epilogue == VCB_EPI_LINEAR1;
    if (head) {
        if (a->hidden <= 0 || a->hidden % 128 || !a->q_scale || !a->k_scale || !a->rope || a->rope_rows <= 0)
            return set_error("gemm: QKV epilogue needs hidden %% 128 == 0, q/k scales and the rope table");
        if (a->epilogue == VCB_EPI_LINEAR1 && (!a->out2 || a->ldo2 % 8 || a->out2_col_offset % 8))
            return set_error("gemm: LINEAR1 epilogue needs out2");
        if (a->epilogue == VCB_EPI_QKV && a->N != 3 * a->hidden) return set_error("gemm: QKV epilogue needs N == 3*hidden");
    }
    if (a->sp_world > 1) {
        if (!head) return set_error("gemm: sp_world > 1 needs the QKV or LINEAR1 epilogue");
        if (a->sp_world > VCB_SP_MAX || a->M != a->rows_per_batch || (a->hidden / 128) % a->sp_world || a->sp_row_offset < 0)
            return set_error("gemm: sequence-parallel routing needs one sample, world <= %d and heads %% world == 0", VCB_SP_MAX);
        for (int r = 0; r < a->sp_world; ++r)
            if (!a->sp_out[r]) return set_error("gemm: sp_out[%d] is null", r);
    }
    if (a->epilogue == VCB_EPI_GATE_RES && (!a->res || a->ld_res % 8 || a->gate_stride % 8))
        return set_error("gemm: GATE_RES epilogue needs res (gate may be NULL = ungated residual)");
    if (a->epilogue < 0 || a->epilogue > VCB_EPI_BIAS_F32) return set_error("gemm: unknown epilogue %d", a->epilogue);
    if (a->rows_per_batch <= 0 || a->M % a->rows_per_batch) return set_error("gemm: M must be a multiple of rows_per_batch");
    const int64_t a_bstride = a->a_batch_stride ? a->a_batch_stride : (int64_t)a->rows_per_batch * a->lda;
    if (a_bstride % 8) return set_error("gemm: a_batch_stride must be a multiple of 8");
    if (a->cta_group < 0 || a->cta_group > 2) return set_error("gemm: cta_group must be 0 (auto), 1 or 2");
    if (a->row_stats) {
        if (a->epilogue != VCB_EPI_GATE_RES) return set_error("gemm: row_stats needs the GATE_RES epilogue");
        if (a->N % 64) return set_error("gemm: row_stats needs N %% 64 == 0");
        if (a->block_n && a->block_n != 128 && a->block_n != 256) return set_error("gemm: row_stats needs block_n 128 or 256");
    }
    if (reinterpret_cast<uintptr_t>(a->bias) & 15) return set_error("gemm: bias must be 16-byte aligned (the epilogue reads it as float4)");
    if (a->operand_dtype != VCB_DTYPE_BF16 && a->operand_dtype != VCB_DTYPE_E4M3) return set_error("gemm: unknown operand_dtype %d", a->operand_dtype);
    if (a->operand_dtype == VCB_DTYPE_E4M3) {
        if (a->lda % 16 || a->ldw % 16 || a_bstride % 16) return set_error("gemm (fp8): lda / ldw / a_batch_stride must be multiples of 16 bytes");
        if (a->sp_world > 1) return set_error("gemm (fp8): the sequence-parallel routing takes bf16 operands");
        if (a->epilogue == VCB_EPI_BIAS_F32) return set_error("gemm (fp8): the fp32-output epilogue is bf16-operand only");
        if (reinterpret_cast<uintptr_t>(a->w_scale) & 15) return set_error("gemm (fp8): w_scale must be 16-byte aligned (read as float4)");
        if (a->block_n && a->block_n != 128 && a->block_n != 256) return set_error("gemm (fp8): block_n must be 128 or 256");
    }
    if (a->lora_rank < 0 || a->lora_rank % 8) return set_error("gemm: lora_rank must be a non-negative multiple of 8 (16-byte rows of T and lora_b)");
    if (a->lora_rank > 0) {
        if (!a->lora_t || !a->lora_b) return set_error("gemm: a LoRA k-tail (lora_rank > 0) needs lora_t and lora_b");
        if (a->operand_dtype == VCB_DTYPE_E4M3) return set_error("gemm (fp8): the LoRA k-tail takes bf16 operands");
        if (a->ld_lora_t % 8 || a->lora_t_batch_stride % 8) return set_error("gemm: ld_lora_t and lora_t_batch_stride must be multiples of 8");
    }
    return 0;
}

int build_problem(const vcb_gemm_args* a, int bn, int cg, Problem* out) {
    const int batch = a->M / a->rows_per_batch;
    const int64_t a_bstride = a->a_batch_stride ? a->a_batch_stride : (int64_t)a->rows_per_batch * a->lda;
    GemmParams& p = out->p;
    p = GemmParams{};
    p.N = a->N; p.K = a->K; p.batch = batch;
    p.rows_per_batch = a->rows_per_batch; p.out_batch_rows = a->out_batch_rows; p.out_row_offset = a->out_row_offset;
    p.bias = a->bias;
    p.out = (__nv_bfloat16*)a->out; p.ldo = a->ldo; p.out_col_offset = a->out_col_offset;
    p.gate = (const __nv_bfloat16*)a->gate; p.gate_stride = a->gate_stride;
    p.res = (const __nv_bfloat16*)a->res; p.ld_res = a->ld_res;
    p.row_stats = a->epilogue == VCB_EPI_GATE_RES ? (float2*)a->row_stats : nullptr;
    p.hidden = a->hidden; p.q_scale = (const __nv_bfloat16*)a->q_scale; p.k_scale = (const __nv_bfloat16*)a->k_scale;
    p.rope = (const float2*)a->rope; p.rope_rows = a->rope_rows;
    p.out2 = (__nv_bfloat16*)a->out2; p.ldo2 = a->ldo2; p.out2_col_offset = a->out2_col_offset;
    p.sp_world = a->sp_world > 1 ? a->sp_world : 0; p.sp_row_offset = a->sp_row_offset;
    p.lora_rank = a->lora_rank; p.alpha = a->alpha;
    const bool fp8 = a->operand_dtype == VCB_DTYPE_E4M3;
    const int eb = fp8 ? 1 : 2;                    // operand bytes per element; a k-block is 128 bytes of K either way
    p.a_scale = fp8 ? a->a_scale : nullptr; p.w_scale = fp8 ? a->w_scale : nullptr;
    for (int r = 0; r < kSpMaxRanks; ++r) p.sp_out[r] = r < p.sp_world ? (__nv_bfloat16*)a->sp_out[r] : nullptr;
    if (int rc = make_tmap_3d(&out->ta, a->A, (uint64_t)a->K, (uint64_t)a->rows_per_batch, (uint64_t)batch, (uint64_t)a->lda,
                              (uint64_t)a_bstride, 128 / eb, 128, eb)) return rc;
    if (int rc = make_tmap_2d(&out->tb, a->W, (uint64_t)a->K, (uint64_t)a->N, (uint64_t)a->ldw, 128 / eb, (uint32_t)(bn / cg), eb)) return rc;
    out->tt = out->ta; out->tl = out->tb;
    if (a->lora_rank > 0) {
        const int64_t t_bstride = a->lora_t_batch_stride ? a->lora_t_batch_stride : (int64_t)a->rows_per_batch * a->ld_lora_t;
        if (int rc = make_tmap_3d(&out->tt, a->lora_t, (uint64_t)a->lora_rank, (uint64_t)a->rows_per_batch, (uint64_t)batch,
                                  (uint64_t)a->ld_lora_t, (uint64_t)t_bstride, 64, 128)) return rc;
        if (int rc = make_tmap_2d(&out->tl, a->lora_b, (uint64_t)a->lora_rank, (uint64_t)a->N, (uint64_t)a->lora_rank, 64, (uint32_t)(bn / cg))) return rc;
    }
    return 0;
}

int gemm_dispatch(const vcb_gemm_args* a, const vcb_gemm_args* a1, void* stream) {
    if (int rc = check_gemm_args(a)) return rc;
    if (a1) {
        if (int rc = check_gemm_args(a1)) return rc;
        if (a1->N != a->N || a1->K != a->K || a1->epilogue != a->epilogue || (a1->sp_world > 1) != (a->sp_world > 1) ||
            a1->operand_dtype != a->operand_dtype || a1->lora_rank != a->lora_rank)
            return set_error("gemm (grouped): both problems need the same N, K, LoRA rank, epilogue, operand dtype and sequence-parallel mode");
    }
    if (int rc = ensure_device()) return rc;
    const bool head = a->epilogue == VCB_EPI_QKV || a->epilogue == VCB_EPI_LINEAR1;
    int cg, bn;
    // tile choice for the combined tile count (the second problem only adds tiles of the same shape)
    const int batch = a->M / a->rows_per_batch;
    float rate;
    const bool fp8 = a->operand_dtype == VCB_DTYPE_E4M3;
    const bool stats = a->row_stats || (a1 && a1->row_stats);      // 64-column statistics slots: tiles of 128 or 256 columns
    pick_tile(batch, a->rows_per_batch + (a1 ? a1->M / batch : 0), a->N, a->K + a->lora_rank, head || fp8 || stats, a->cta_group ? a->cta_group : forced_cta_group(),
              a->block_n, &cg, &bn, &rate);
    ProfScope prof(PROF_GEMM, stream, a->M + (a1 ? a1->M : 0), a->N, a->K, a->epilogue | ((bn >> 5) << 8) | (cg << 16));
    Problem g0, g1;
    if (int rc = build_problem(a, bn, cg, &g0)) return rc;
    if (a1) {
        if (int rc = build_problem(a1, bn, cg, &g1)) return rc;
    } else {
        g1 = g0;
        g1.p = GemmParams{};            // batch == 0: no second problem
    }
    // tile raster: M-fastest.  VCB_GEMM_RASTER=1 selects the N-fastest alternative (a wave = a band of A rows x all weight tiles,
    // A evict-first, B evict-last) for A/B runs and tests.
    {
        static const int forced = [] { const char* e = getenv("VCB_GEMM_RASTER"); return e ? atoi(e) : -1; }();
        const int nf = forced > 0 ? 1 : 0;
        g0.p.n_fastest = nf;
        g1.p.n_fastest = nf;
    }
    cudaStream_t st = (cudaStream_t)stream;
    if (fp8) {
#define VCB_GEMM_CASE8(BN, CG) \
    if (bn == BN && cg == CG) return launch_gemm_epi_fp8<BN, CG>(a->epilogue, g0, g1, rate, st);
        VCB_GEMM_CASE8(128, 1)
        VCB_GEMM_CASE8(256, 1)
        VCB_GEMM_CASE8(128, 2)
        VCB_GEMM_CASE8(256, 2)
#undef VCB_GEMM_CASE8
        return set_error("gemm (fp8): unsupported (block_n=%d, cta_group=%d)", bn, cg);
    }
#define VCB_GEMM_CASE(BN, CG) \
    if (bn == BN && cg == CG) return launch_gemm_epi<BN, CG>(a->epilogue, g0, g1, rate, st);
    VCB_GEMM_CASE(64, 1)
    VCB_GEMM_CASE(128, 1)
    VCB_GEMM_CASE(192, 1)
    VCB_GEMM_CASE(256, 1)
    VCB_GEMM_CASE(128, 2)
    VCB_GEMM_CASE(192, 2)
    VCB_GEMM_CASE(256, 2)
#undef VCB_GEMM_CASE
    return set_error("gemm: unsupported (block_n=%d, cta_group=%d)", bn, cg);
}

}  // namespace

extern "C" int vcb_gemm_bf16(const vcb_gemm_args* a, void* stream) { return gemm_dispatch(a, nullptr, stream); }

extern "C" int vcb_gemm_bf16_grouped(const vcb_gemm_args* a0, const vcb_gemm_args* a1, void* stream) {
    if (!a1) return set_error("gemm (grouped): second problem is null");
    return gemm_dispatch(a0, a1, stream);
}

// ------------------------------------------------------------------------------------------------
// 3x3 convolution, NHWC, stride 1, zero padding 1: implicit GEMM on the same wgmma kernel (A_CONV3X3)
// ------------------------------------------------------------------------------------------------
namespace {
template <int BN, int EPI>
int launch_conv_inst(const CUtensorMap& ta, const CUtensorMap& tb, const GemmParams& p, cudaStream_t st) {
    using Cfg = GemmCfg<BN, 1>;
    auto kern = gemm_wgmma_kernel<BN, 1, EPI, A_CONV3X3>;
    static std::once_flag once;
    static cudaError_t attr_err = cudaSuccess;
    std::call_once(once, [&] {
        attr_err = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmemBytes);
    });
    if (attr_err != cudaSuccess) return set_error("cudaFuncSetAttribute(conv): %s", cudaGetErrorString(attr_err));
    const int tiles = p.batch * ((p.conv_W + kConvTileW - 1) / kConvTileW) * ((p.conv_H + kConvTileH - 1) / kConvTileH) *
                      ((p.N + BN - 1) / BN);
    int grid = num_sms();
    if (tiles < grid) grid = tiles;
    GemmParams none{};
    cudaError_t e = launch_pdl(kern, dim3(grid), dim3(kGemmThreads), (size_t)Cfg::kSmemBytes, st, 1, ta, tb, p, ta, tb, none, StreamKParams{nullptr, nullptr, 0, 0},
                               ta, tb, ta, tb);
    if (e != cudaSuccess) return set_error("conv3x3 launch: %s", cudaGetErrorString(e));
    count_launch();
    return 0;
}
}  // namespace

extern "C" int vcb_conv3x3_nhwc(const void* x, const void* w, const float* bias, const void* res, void* out, int32_t n,
                                int32_t H, int32_t W, int32_t cin, int32_t cout, int32_t stride, void* stream) {
    if (!x || !w || !out || n <= 0 || H <= 0 || W <= 0) return set_error("conv3x3: bad arguments");
    if (stride != 1 && stride != 2) return set_error("conv3x3: stride must be 1 or 2");
    if (stride == 2 && ((H | W) & 1)) return set_error("conv3x3: stride 2 needs even H and W");
    const int Ho = H / stride, Wo = W / stride;
    if (cin % 64 || cout % 8) return set_error("conv3x3: Cin must be a multiple of 64 and Cout of 8 (pad the weights)");
    if (int rc = ensure_device()) return rc;
    ProfScope prof(PROF_CONV, stream, n * Ho * Wo, cout, 9 * cin, stride);
    GemmParams p{};
    p.N = cout; p.K = 9 * cin; p.batch = n;
    p.rows_per_batch = Ho * Wo; p.out_batch_rows = Ho * Wo; p.out_row_offset = 0;
    p.bias = bias; p.out = (__nv_bfloat16*)out; p.ldo = cout;
    p.res = (const __nv_bfloat16*)res; p.ld_res = cout;
    p.conv_H = Ho; p.conv_W = Wo; p.conv_C = cin; p.conv_stride = stride;
    const int bn = cout >= 256 ? 256 : (cout >= 128 ? 128 : 64);
    CUtensorMap ta, tb;
    const uint64_t dims[4] = {(uint64_t)cin, (uint64_t)W, (uint64_t)H, (uint64_t)n};
    const uint64_t str[3] = {(uint64_t)cin, (uint64_t)W * cin, (uint64_t)H * W * cin};
    const uint32_t box[4] = {64, (uint32_t)(kConvTileW * stride), (uint32_t)(kConvTileH * stride), 1};
    const uint32_t estr[4] = {1, (uint32_t)stride, (uint32_t)stride, 1};
    if (int rc = make_tmap_4d(&ta, x, dims, str, box, estr)) return rc;
    if (int rc = make_tmap_2d(&tb, w, (uint64_t)9 * cin, (uint64_t)cout, (uint64_t)9 * cin, 64, (uint32_t)bn)) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    const bool r = res != nullptr;
    if (bn == 256) return r ? launch_conv_inst<256, EPI_GATE_RES>(ta, tb, p, st) : launch_conv_inst<256, EPI_BIAS>(ta, tb, p, st);
    if (bn == 128) return r ? launch_conv_inst<128, EPI_GATE_RES>(ta, tb, p, st) : launch_conv_inst<128, EPI_BIAS>(ta, tb, p, st);
    return r ? launch_conv_inst<64, EPI_GATE_RES>(ta, tb, p, st) : launch_conv_inst<64, EPI_BIAS>(ta, tb, p, st);
}

// ------------------------------------------------------------------------------------------------
// attention
// ------------------------------------------------------------------------------------------------
namespace {
// workspace of the persistent attention schedule: one (O, l, m) slot and one flag per CTA, per stream; allocated on
// first use (call once before CUDA-graph capture)
struct AttnScratch { float* ws = nullptr; int* flags = nullptr; int epoch = 0; unsigned long long* timeline = nullptr; int last_grid = 0; };
AttnScratch* g_last_attn_scratch = nullptr;       // debug: the scratch of the most recent persistent launch (vcb_debug_attn4_timeline)
inline AttnScratch* attn_scratch(cudaStream_t st) {
    static std::mutex mu;
    static std::map<cudaStream_t, AttnScratch> pool;
    std::lock_guard<std::mutex> lk(mu);
    AttnScratch& s = pool[st];
    if (!s.ws) {
        const size_t n = 160;                                  // >= number of SMs
        if (cudaMalloc(&s.ws, n * kAttn4SlotFloats * sizeof(float)) != cudaSuccess) return nullptr;
        if (cudaMalloc(&s.flags, n * sizeof(int)) != cudaSuccess) return nullptr;
        cudaMemset(s.flags, 0, n * sizeof(int));
        static const bool tl = [] { const char* e = getenv("VCB_ATTN4_TIMELINE"); return e && atoi(e); }();
        if (tl && cudaMalloc(&s.timeline, n * (kAttn4MaxSegs + 2) * sizeof(unsigned long long)) != cudaSuccess) s.timeline = nullptr;
    }
    return &s;
}
// What VCB_ATTN_SCHED_AUTO resolves to.  Default: one CTA per query tile; VCB_ATTN_PERSIST=1 makes AUTO pick the persistent
// schedule (tools/bench_attn_quick.py compares the two).
inline int attn_persist_mode() {
    static const int m = [] { const char* e = getenv("VCB_ATTN_PERSIST"); return (e && atoi(e)) ? 1 : 0; }();
    return m;
}

int attention_launch(const void* qkv, int64_t ld_qkv, int32_t q_col, int32_t k_col, int32_t v_col,
                     const int32_t* seqlens, int32_t B, int32_t L, int32_t heads, void* out, int64_t ldo,
                     int32_t out_col_offset, void* const* out_peers, int32_t world, int32_t rows_per_rank, float bound, int32_t schedule,
                     void* stream) {
    if (schedule < VCB_ATTN_SCHED_AUTO || schedule > VCB_ATTN_SCHED_PERSISTENT) return set_error("attention: unknown schedule %d", schedule);
    if (bound < 0.f || bound > 64.f) return set_error("attention: score_bound_log2 must be in [0, 64] (0 = exact online softmax)");
    if (!qkv || (!out && !out_peers) || B <= 0 || L <= 0 || heads <= 0) return set_error("attention: bad arguments");
    if (ld_qkv % 8 || ldo % 8 || q_col % 8 || k_col % 8 || v_col % 8 || out_col_offset % 8)
        return set_error("attention: leading dims / column offsets must be multiples of 8");
    if (int rc = ensure_device()) return rc;
    static std::once_flag once;
    static cudaError_t attr_err = cudaSuccess;
    std::call_once(once, [&] {
        attr_err = cudaFuncSetAttribute(attn_fwd_wgmma_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, kAttnSmemBytes);
        if (attr_err == cudaSuccess)
            attr_err = cudaFuncSetAttribute(attn_fwd_wgmma_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, kAttnSmemBytes);
    });
    if (attr_err != cudaSuccess) return set_error("cudaFuncSetAttribute(attn): %s", cudaGetErrorString(attr_err));
    CUtensorMap tm;
    if (int rc = make_tmap_3d(&tm, qkv, (uint64_t)ld_qkv, (uint64_t)L, (uint64_t)B, (uint64_t)ld_qkv, (uint64_t)ld_qkv * L, 64, 128)) return rc;
    AttnParams p{};
    p.B = B; p.L = L; p.H = heads; p.seqlens = seqlens;
    p.out = (__nv_bfloat16*)out; p.ldo = ldo; p.out_col_offset = out_col_offset;
    p.q_col = q_col; p.k_col = k_col; p.v_col = v_col;
    p.scale_log2 = 0.08838834764831845f * 1.4426950408889634f;     // 128^-0.5 * log2(e)
    static const bool no_bound = [] { const char* e = getenv("VCB_ATTN_EXACT_MAX"); return e && atoi(e); }();
    const bool fixed = bound > 0.f && !no_bound;
    p.fixed_max = fixed ? bound : 0.f;
    if (out_peers) {
        if (world < 2 || world > VCB_SP_MAX || B != 1 || seqlens || rows_per_rank <= 0 || (int64_t)rows_per_rank * world != L)
            return set_error("attention (sp): needs one unpadded sample with L == world * rows_per_rank, 2 <= world <= %d", VCB_SP_MAX);
        p.sp_world = world; p.sp_rows = rows_per_rank;
        for (int r = 0; r < world; ++r) {
            if (!out_peers[r]) return set_error("attention (sp): out_peers[%d] is null", r);
            p.sp_out[r] = (__nv_bfloat16*)out_peers[r];
        }
    }
    ProfScope prof(PROF_ATTN, stream, B, L, heads, fixed ? 1 : 0);
    // Persistent schedule: unpadded batches with enough (query tile x key tile) work to give every SM a share of at least a few
    // key tiles; right-padded batches stay on the per-tile grid.
    const long long n_qt = (L + kAttnTile - 1) / kAttnTile;
    const long long n_units = (long long)B * heads * n_qt, total_steps = n_units * n_qt;
    int pgrid = num_sms();
    if (total_steps / pgrid < 4) pgrid = (int)(total_steps / 4 > 0 ? total_steps / 4 : 1);   // tiny problems: >= 4 key-tile steps per CTA
    // a CTA's segment list: one entry per full round + the pieces of its tail share; beyond the kernel's capacity (huge batches of
    // short sequences) use the per-tile grid.
    // Sequence-parallel routing (O rows leave through the peer-mapped pointers in either schedule): few heads per rank leave the
    // per-tile grid below one wave, and the key-tile split then fills the idle SMs; it costs a partial dump, a fold and a phase
    // hand-over per launch (tools/attn4_timeline.py), so AUTO takes it only when the per-tile grid would fill < 40 % of the SMs.
    // VCB_SP_ATTN_PERSIST=0 / 1 forces it off / on.
    static const int sp_persist_env = [] { const char* e = getenv("VCB_SP_ATTN_PERSIST"); return e ? (atoi(e) ? 1 : 0) : -1; }();
    const bool sp_persist = out_peers && (sp_persist_env >= 0 ? sp_persist_env == 1 : n_units * 10 < (long long)num_sms() * 4);
    const bool persist_ok = !seqlens && (!out_peers || sp_persist) && num_sms() <= 160 && n_units / pgrid + 4 <= kAttn4MaxSegs;
    if (schedule == VCB_ATTN_SCHED_PERSISTENT && !persist_ok)
        return set_error("attention: the persistent schedule takes unpadded batches (seqlens == NULL), no sequence-parallel routing");
    AttnSkParams skp{nullptr, nullptr, 0, 0, nullptr};
    dim3 grid((unsigned)n_qt, heads, B);
    if (persist_ok && (schedule == VCB_ATTN_SCHED_PERSISTENT || (schedule == VCB_ATTN_SCHED_AUTO && (attn_persist_mode() != 0 || sp_persist)))) {
        grid = dim3(pgrid);
        prof.set_info(3, (fixed ? 1 : 0) | 2);
        AttnScratch* sc = attn_scratch((cudaStream_t)stream);
        if (!sc) return set_error("attention: workspace allocation failed");
        static const int no_split = [] { const char* e = getenv("VCB_ATTN4_NOSPLIT"); return (e && atoi(e)) ? 1 : 0; }();
        skp = AttnSkParams{sc->ws, sc->flags, ++sc->epoch, no_split, sc->timeline};
        if (sc->timeline) cudaMemsetAsync(sc->timeline, 0, 160 * (kAttn4MaxSegs + 2) * sizeof(unsigned long long), (cudaStream_t)stream);
        sc->last_grid = pgrid;
        g_last_attn_scratch = sc;
    }
    cudaError_t e = fixed ? launch_pdl(attn_fwd_wgmma_kernel<true>, grid, dim3(kAttnThreads), (size_t)kAttnSmemBytes, (cudaStream_t)stream, 1, tm, p, skp)
                          : launch_pdl(attn_fwd_wgmma_kernel<false>, grid, dim3(kAttnThreads), (size_t)kAttnSmemBytes, (cudaStream_t)stream, 1, tm, p, skp);
    if (e != cudaSuccess) return set_error("attention launch: %s", cudaGetErrorString(e));
    count_launch();
    return 0;
}
}  // namespace

// debug (VCB_ATTN4_TIMELINE=1): per-CTA globaltimer stamps of the most recent persistent attention launch -- [grid][kAttn4MaxSegs + 2]
// = start, end of every segment (0 = unused).  Synchronises the device.  Returns the grid size, or -1.
extern "C" int vcb_debug_attn4_timeline(unsigned long long* out, int32_t capacity) {
    AttnScratch* sc = g_last_attn_scratch;
    if (!sc || !sc->timeline || !out) return -1;
    cudaDeviceSynchronize();
    const int n = sc->last_grid * (kAttn4MaxSegs + 2);
    if (capacity < n) return -1;
    if (cudaMemcpy(out, sc->timeline, (size_t)n * sizeof(unsigned long long), cudaMemcpyDeviceToHost) != cudaSuccess) return -1;
    return sc->last_grid;
}

extern "C" int vcb_attention_fwd(const void* qkv, int64_t ld_qkv, int32_t q_col, int32_t k_col, int32_t v_col,
                                 const int32_t* seqlens, int32_t B, int32_t L, int32_t heads, void* out, int64_t ldo,
                                 int32_t out_col_offset, void* stream) {
    if (!out) return set_error("attention: bad arguments");
    return attention_launch(qkv, ld_qkv, q_col, k_col, v_col, seqlens, B, L, heads, out, ldo, out_col_offset, nullptr, 0, 0, 0.f,
                            VCB_ATTN_SCHED_AUTO, stream);
}

extern "C" int vcb_attention_fwd_ex(const vcb_attn_args* a, void* stream) {
    if (!a) return set_error("attention: null args");
    if (!a->out_peers && !a->out) return set_error("attention: bad arguments");
    return attention_launch(a->qkv, a->ld_qkv, a->q_col, a->k_col, a->v_col, a->seqlens, a->out_peers ? 1 : a->B, a->L, a->heads, a->out,
                            a->ldo, a->out_col_offset, a->out_peers, a->world, a->rows_per_rank, a->score_bound_log2, a->schedule, stream);
}

extern "C" int vcb_attention_fwd_sp(const void* qkv, int64_t ld_qkv, int32_t q_col, int32_t k_col, int32_t v_col, int32_t L,
                                    int32_t heads, void* const* out_peers, int32_t world, int32_t rows_per_rank, int64_t ldo,
                                    int32_t out_col_offset, void* stream) {
    if (!out_peers) return set_error("attention (sp): out_peers is null");
    return attention_launch(qkv, ld_qkv, q_col, k_col, v_col, nullptr, 1, L, heads, nullptr, ldo, out_col_offset, out_peers, world,
                            rows_per_rank, 0.f, VCB_ATTN_SCHED_AUTO, stream);
}

// ------------------------------------------------------------------------------------------------
// sequence-parallel plumbing: peer-mappable allocations (CUDA IPC) and the cross-GPU phase barrier
// ------------------------------------------------------------------------------------------------
static_assert(sizeof(cudaIpcMemHandle_t) == 64, "vcb_peer_alloc hands out 64-byte handles");

extern "C" int vcb_peer_alloc(int64_t bytes, void** ptr, void* handle64) {
    if (bytes <= 0 || !ptr || !handle64) return set_error("peer_alloc: bad arguments");
    if (int rc = ensure_device()) return rc;
    void* d = nullptr;
    cudaError_t e = cudaMalloc(&d, (size_t)bytes);
    if (e != cudaSuccess) return set_error("peer_alloc: cudaMalloc(%lld): %s", (long long)bytes, cudaGetErrorString(e));
    e = cudaMemset(d, 0, (size_t)bytes);                  // flag arrays must start at zero; synchronous on return
    if (e == cudaSuccess) e = cudaDeviceSynchronize();
    if (e != cudaSuccess) {
        cudaFree(d);
        return set_error("peer_alloc: cudaMemset: %s", cudaGetErrorString(e));
    }
    cudaIpcMemHandle_t h;
    e = cudaIpcGetMemHandle(&h, d);
    if (e != cudaSuccess) {
        cudaFree(d);
        return set_error("peer_alloc: cudaIpcGetMemHandle: %s", cudaGetErrorString(e));
    }
    memcpy(handle64, &h, 64);
    *ptr = d;
    return 0;
}

extern "C" int vcb_peer_open(const void* handle64, void** ptr) {
    if (!handle64 || !ptr) return set_error("peer_open: bad arguments");
    if (int rc = ensure_device()) return rc;
    cudaIpcMemHandle_t h;
    memcpy(&h, handle64, 64);
    void* d = nullptr;
    cudaError_t e = cudaIpcOpenMemHandle(&d, h, cudaIpcMemLazyEnablePeerAccess);
    if (e != cudaSuccess) return set_error("peer_open: cudaIpcOpenMemHandle: %s (peer access between the two GPUs is required)", cudaGetErrorString(e));
    *ptr = d;
    return 0;
}

extern "C" int vcb_peer_close(void* ptr) {
    if (!ptr) return 0;
    cudaError_t e = cudaIpcCloseMemHandle(ptr);
    return e == cudaSuccess ? 0 : set_error("peer_close: %s", cudaGetErrorString(e));
}

extern "C" int vcb_peer_free(void* ptr) {
    if (!ptr) return 0;
    cudaError_t e = cudaFree(ptr);
    return e == cudaSuccess ? 0 : set_error("peer_free: %s", cudaGetErrorString(e));
}

extern "C" int vcb_sp_barrier(int32_t* const* flags, int32_t world, int32_t rank, int32_t epoch, int32_t* err, int32_t timeout_ms,
                              void* stream) {
    if (!flags || !err || world < 1 || world > VCB_SP_MAX || rank < 0 || rank >= world) return set_error("sp_barrier: bad arguments");
    if (int rc = ensure_device()) return rc;
    SpFlags f{};
    for (int r = 0; r < world; ++r) {
        if (!flags[r]) return set_error("sp_barrier: flags[%d] is null", r);
        f.f[r] = flags[r];
    }
    ProfScope prof(PROF_OTHER, stream);
    cudaError_t e = launch_pdl(sp_barrier_kernel, dim3(1), dim3(32), (size_t)0, (cudaStream_t)stream, 1, f, (int)world, (int)rank, (int)epoch,
                               (int*)err, (unsigned long long)(timeout_ms > 0 ? timeout_ms : 2000) * 1000000ull);
    if (e != cudaSuccess) return set_error("sp_barrier launch: %s", cudaGetErrorString(e));
    count_launch();
    return 0;
}

// ------------------------------------------------------------------------------------------------
// elementwise
// ------------------------------------------------------------------------------------------------
namespace {
// One AdaLN LayerNorm launch (elementwise.cuh) for the five entry points below: one or two problems (a1 may be NULL), e4m3
// output with per-row scales when fp8, statistics from the producing GEMM when with_stats.  `fn` prefixes the error messages.
int ln_launch(const char* fn, const vcb_ln_args* a0, const vcb_ln_args* a1, bool fp8, float* row_scale0, float* row_scale1,
              bool with_stats, const void* stats0, const void* stats1, int32_t n_slots, int64_t ldx, int64_t ldy, int64_t mod_stride,
              int32_t hidden, int32_t batch_rows, void* stream) {
    if (!a0) return set_error("%s: null problem", fn);
    if (hidden % 256 || hidden > kLnMaxHidden) return set_error("%s: hidden must be a multiple of 256, <= %d", fn, kLnMaxHidden);
    if (ldx % 8 || mod_stride % 8 || ldy % (fp8 ? 16 : 8))
        return set_error("%s: ldx / mod_stride must be multiples of 8, the output stride of %d", fn, fp8 ? 16 : 8);
    if (with_stats && n_slots <= 0) return set_error("%s: n_slots must be positive", fn);
    const vcb_ln_args* a[2] = {a0, a1};
    float* rs[2] = {row_scale0, row_scale1};
    const void* st[2] = {stats0, stats1};
    LnProblem p[2] = {};
    for (int i = 0; i < 2; ++i) {
        if (!a[i]) continue;
        if (!a[i]->x || !a[i]->y || !a[i]->shift || !a[i]->scale || a[i]->rows <= 0 || a[i]->rows_per_batch <= 0)
            return set_error("%s: bad arguments", fn);
        if (fp8 && !rs[i]) return set_error("%s: null row_scale", fn);
        if (with_stats && !st[i]) return set_error("%s: null stats", fn);
        p[i] = LnProblem{(const __nv_bfloat16*)a[i]->x, a[i]->y, rs[i], (const float2*)st[i], (const __nv_bfloat16*)a[i]->shift,
                         (const __nv_bfloat16*)a[i]->scale, a[i]->rows, a[i]->rows_per_batch, (a[i]->rows + kLnWarps - 1) / kLnWarps};
    }
    if (batch_rows <= 0) return set_error("%s: batch_rows (rows of one sample in the joint buffer) is required", fn);
    if (int rc = ensure_device()) return rc;
    ProfScope prof(PROF_LN, stream);
    auto kern = fp8 ? (with_stats ? ln_modulate_fp8_stats_kernel : ln_modulate_fp8_kernel)
                    : (with_stats ? ln_modulate_stats_kernel : ln_modulate2_kernel);
    cudaError_t e = launch_pdl(kern, dim3(p[0].blocks + p[1].blocks), dim3(kLnWarps * 32), (size_t)hidden * 8, (cudaStream_t)stream, 1,
                               p[0], p[1], (long long)ldx, (long long)ldy, (long long)mod_stride, (int)hidden, (int)batch_rows, (int)n_slots);
    if (e != cudaSuccess) return set_error("%s launch: %s", fn, cudaGetErrorString(e));
    count_launch();
    return 0;
}
}  // namespace

extern "C" int vcb_ln_modulate(const void* x, int64_t ldx, void* y, int64_t ldy, const void* shift, const void* scale,
                               int64_t mod_stride, int32_t rows, int32_t hidden, int32_t rows_per_batch, int32_t batch_rows,
                               void* stream) {
    const vcb_ln_args a{x, y, shift, scale, rows, rows_per_batch};
    return ln_launch("ln_modulate", &a, nullptr, false, nullptr, nullptr, false, nullptr, nullptr, 0, ldx, ldy, mod_stride, hidden,
                     batch_rows > 0 ? batch_rows : rows_per_batch, stream);
}

extern "C" int vcb_ln_modulate_grouped(const vcb_ln_args* a0, const vcb_ln_args* a1, int64_t ldx, int64_t ldy, int64_t mod_stride,
                                       int32_t hidden, int32_t batch_rows, void* stream) {
    return ln_launch("ln_modulate_grouped", a0, a1, false, nullptr, nullptr, false, nullptr, nullptr, 0, ldx, ldy, mod_stride, hidden,
                     batch_rows, stream);
}

extern "C" int vcb_ln_modulate_stats(const vcb_ln_args* a0, const vcb_ln_args* a1, const void* stats0, const void* stats1, int32_t n_slots,
                                     int64_t ldx, int64_t ldy, int64_t mod_stride, int32_t hidden, int32_t batch_rows, void* stream) {
    return ln_launch("ln_modulate_stats", a0, a1, false, nullptr, nullptr, true, stats0, stats1, n_slots, ldx, ldy, mod_stride, hidden,
                     batch_rows, stream);
}

extern "C" int vcb_ln_modulate_fp8(const vcb_ln_args* a0, const vcb_ln_args* a1, float* row_scale0, float* row_scale1, int64_t ldx,
                                   int64_t ld8, int64_t mod_stride, int32_t hidden, int32_t batch_rows, void* stream) {
    return ln_launch("ln_modulate_fp8", a0, a1, true, row_scale0, row_scale1, false, nullptr, nullptr, 0, ldx, ld8, mod_stride, hidden,
                     batch_rows, stream);
}

extern "C" int vcb_ln_modulate_fp8_stats(const vcb_ln_args* a0, const vcb_ln_args* a1, float* row_scale0, float* row_scale1, const void* stats0,
                                         const void* stats1, int32_t n_slots, int64_t ldx, int64_t ld8, int64_t mod_stride, int32_t hidden,
                                         int32_t batch_rows, void* stream) {
    return ln_launch("ln_modulate_fp8_stats", a0, a1, true, row_scale0, row_scale1, true, stats0, stats1, n_slots, ldx, ld8, mod_stride,
                     hidden, batch_rows, stream);
}

extern "C" int vcb_quantize_rows_e4m3(const void* x, int64_t ldx, void* y8, int64_t ld8, float* row_scale, int64_t rows, int32_t K,
                                      void* stream) {
    if (!x || !y8 || !row_scale) return set_error("quantize_rows_e4m3: null argument");
    if (rows <= 0 || rows > 0x7fffffffLL || K <= 0 || K % 8 || K > kQuantThreads * kQuantMaxChunks * 8)
        return set_error("quantize_rows_e4m3: need rows > 0 and K a multiple of 8, <= %d", kQuantThreads * kQuantMaxChunks * 8);
    if (ldx % 8 || ld8 % 8 || (reinterpret_cast<uintptr_t>(x) & 15) || (reinterpret_cast<uintptr_t>(y8) & 7))
        return set_error("quantize_rows_e4m3: ldx / ld8 must be multiples of 8 elements, x 16-byte and y8 8-byte aligned");
    if (int rc = ensure_device()) return rc;
    ProfScope prof(PROF_OTHER, stream);
    cudaError_t e = launch_pdl(quantize_rows_e4m3_kernel, dim3((unsigned)rows), dim3(kQuantThreads), (size_t)0, (cudaStream_t)stream, 1,
                               (const __nv_bfloat16*)x, (long long)ldx, (uint8_t*)y8, (long long)ld8, row_scale, (int)K);
    if (e != cudaSuccess) return set_error("quantize_rows_e4m3 launch: %s", cudaGetErrorString(e));
    count_launch();
    return 0;
}

extern "C" int vcb_timestep_embedding(const float* t_scaled, const float* freqs, void* out, int32_t n, void* stream) {
    if (!t_scaled || !freqs || !out || n <= 0) return set_error("timestep_embedding: bad arguments");
    if (int rc = ensure_device()) return rc;
    ProfScope prof(PROF_OTHER, stream);
    timestep_embedding_kernel<<<(n * 128 + 127) / 128, 128, 0, (cudaStream_t)stream>>>(t_scaled, freqs, (__nv_bfloat16*)out, n);
    return check_launch("timestep_embedding");
}

extern "C" int vcb_silu(const void* x, void* y, int64_t n, void* stream) {
    if (!x || !y || n <= 0 || n % 2) return set_error("silu: bad arguments");
    if (int rc = ensure_device()) return rc;
    const long long thr = n / 2;
    ProfScope prof(PROF_OTHER, stream);
    silu_kernel<<<(unsigned)((thr + 255) / 256), 256, 0, (cudaStream_t)stream>>>((const __nv_bfloat16*)x, (__nv_bfloat16*)y, n);
    return check_launch("silu");
}

extern "C" int vcb_add3(const void* a, const void* b, int32_t b_rows, const void* c, int32_t c_rows, void* out,
                        int32_t rows, int32_t hidden, void* stream) {
    if (!a || !out || rows <= 0 || hidden <= 0) return set_error("add3: bad arguments");
    if ((b && b_rows <= 0) || (c && c_rows <= 0)) return set_error("add3: bad row counts");
    if (int rc = ensure_device()) return rc;
    const long long n = (long long)rows * hidden;
    ProfScope prof(PROF_OTHER, stream);
    add3_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
        (const __nv_bfloat16*)a, (const __nv_bfloat16*)b, b_rows > 0 ? b_rows : 1, (const __nv_bfloat16*)c,
        c_rows > 0 ? c_rows : 1, (__nv_bfloat16*)out, rows, hidden);
    return check_launch("add3");
}

extern "C" int vcb_rope_table(const float* ids, void* out, int32_t rows, int32_t d0, int32_t d1, int32_t d2, double theta,
                              void* stream) {
    if (!ids || !out || rows <= 0) return set_error("rope_table: bad arguments");
    if (d0 + d1 + d2 != 128 || d0 % 2 || d1 % 2 || d2 % 2) return set_error("rope_table: axes must be even and sum to 128");
    if (int rc = ensure_device()) return rc;
    const int n = rows * 64;
    ProfScope prof(PROF_OTHER, stream);
    rope_table_kernel<<<(n + 255) / 256, 256, 0, (cudaStream_t)stream>>>(ids, (float2*)out, rows, d0, d1, d2, theta);
    return check_launch("rope_table");
}

// One launcher for every ODE stage form (elementwise.cuh, ode_stage_kernel): 16-byte accesses when the layout allows them.
static int ode_launch(const char* name, int form, const void* y0, const void* const* v, int n_v, float h, void* y_out,
                      void* model_in, int64_t ld_in, int64_t rows, int32_t C, void* stream) {
    if (!y0 || !y_out || rows <= 0 || C <= 0) return set_error("%s: bad arguments", name);
    if (model_in && ld_in < C) return set_error("%s: ld_in (%lld) < C (%d)", name, (long long)ld_in, C);
    OdeVs vs{};
    uintptr_t addr_bits = (uintptr_t)y0 | (uintptr_t)y_out | (uintptr_t)model_in;
    for (int i = 0; i < n_v; ++i) {
        if (!v[i]) return set_error("%s: v[%d] is NULL", name, i);
        vs.v[i] = (const __nv_bfloat16*)v[i];
        addr_bits |= (uintptr_t)v[i];
    }
    if (int rc = ensure_device()) return rc;
    const bool vec = C % 8 == 0 && (!model_in || ld_in % 8 == 0) && addr_bits % 16 == 0;
    const long long threads = rows * C / (vec ? 8 : 1);
    const unsigned grid = (unsigned)((threads + 255) / 256);
    const auto* y0b = (const __nv_bfloat16*)y0;
    auto* yo = (__nv_bfloat16*)y_out;
    auto* mi = (__nv_bfloat16*)model_in;
    cudaStream_t st = (cudaStream_t)stream;
    ProfScope prof(PROF_OTHER, stream);
#define VCB_ODE_CASE(F)                                                                                   \
    case F:                                                                                               \
        if (vec) ode_stage_kernel<F, 8><<<grid, 256, 0, st>>>(y0b, vs, h, yo, mi, ld_in, rows, C);         \
        else ode_stage_kernel<F, 1><<<grid, 256, 0, st>>>(y0b, vs, h, yo, mi, ld_in, rows, C);             \
        break;
    switch (form) {
        VCB_ODE_CASE(kOdeAxpy)
        VCB_ODE_CASE(kOdeRk4K2)
        VCB_ODE_CASE(kOdeRk4K3)
        VCB_ODE_CASE(kOdeRk4K4)
        VCB_ODE_CASE(kOdeRk4Final)
        default: return set_error("%s: bad stage form %d", name, form);
    }
#undef VCB_ODE_CASE
    return check_launch(name);
}

static float bf16_round_host(float x) { return __bfloat162float(__float2bfloat16_rn(x)); }

extern "C" int vcb_euler_update(const void* x, const void* v, float dt_bf16, void* x_new, void* model_in, int64_t ld_in,
                                int64_t rows, int32_t C, void* stream) {
    if (!v) return set_error("euler_update: bad arguments");
    return ode_launch("euler_update", kOdeAxpy, x, &v, 1, dt_bf16, x_new, model_in, ld_in, rows, C, stream);
}

extern "C" int vcb_ode_stage(int32_t method, int32_t stage, const void* y0, const void* const* v, int32_t n_v, float dt,
                             void* y_out, void* model_in, int64_t ld_in, int64_t rows, int32_t C, void* stream) {
    static const int kForms[3][4] = {{kOdeAxpy, -1, -1, -1},
                                     {kOdeAxpy, kOdeAxpy, -1, -1},
                                     {kOdeRk4K2, kOdeRk4K3, kOdeRk4K4, kOdeRk4Final}};
    if (method < VCB_ODE_EULER || method > VCB_ODE_RK4) return set_error("ode_stage: unknown method %d", method);
    if (stage < 0 || stage > 3 || kForms[method][stage] < 0) return set_error("ode_stage: method %d has no stage %d", method, stage);
    if (!v || n_v != stage + 1) return set_error("ode_stage: stage %d takes the %d model outputs v_1..v_%d, got n_v = %d", stage,
                                                 stage + 1, stage + 1, n_v);
    // midpoint: the state y0 + k1 * half_dt scales by the fp32 tensor 0.5 * dt, the final update y0 + dt * k2 reads only k2
    const float h = bf16_round_host(method == VCB_ODE_MIDPOINT && stage == 0 ? 0.5f * dt : dt);
    const void* const* vv = method == VCB_ODE_MIDPOINT && stage == 1 ? v + 1 : v;
    const int nv = method == VCB_ODE_MIDPOINT && stage == 1 ? 1 : n_v;
    return ode_launch("ode_stage", kForms[method][stage], y0, vv, nv, h, y_out, model_in, ld_in, rows, C, stream);
}

extern "C" int vcb_copy_cols(const void* src, int64_t lds, void* dst, int64_t ldd, int32_t col0, int64_t rows, int32_t C,
                             void* stream) {
    if (!src || !dst || rows <= 0 || C <= 0) return set_error("copy_cols: bad arguments");
    if (int rc = ensure_device()) return rc;
    const long long n = rows * C;
    ProfScope prof(PROF_OTHER, stream);
    copy_cols_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
        (const __nv_bfloat16*)src, lds, (__nv_bfloat16*)dst, ldd, col0, rows, C);
    return check_launch("copy_cols");
}

// ------------------------------------------------------------------------------------------------
// probe
// ------------------------------------------------------------------------------------------------
extern "C" int vcb_debug_umma_probe(const void* a, const void* b, float* out, int32_t ksteps, int32_t b_mn_major,
                                    int32_t a_from_regs, uint32_t b_lbo, uint32_t b_sbo, uint32_t b_kstep_bytes,
                                    void* stream) {
    if (!a || !b || !out || (ksteps != 4 && ksteps != 8)) return set_error("probe: ksteps must be 4 or 8");
    if (int rc = ensure_device()) return rc;
    const int K = 16 * ksteps;
    static std::once_flag once;
    std::call_once(once, [&] { cudaFuncSetAttribute(wgmma_probe_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 67 * 1024); });
    CUtensorMap ta, tb;
    if (int rc = make_tmap_2d(&ta, a, (uint64_t)K, 128, (uint64_t)K, 64, 128)) return rc;
    if (b_mn_major) {
        if (int rc = make_tmap_2d(&tb, b, 128, (uint64_t)K, 128, 64, (uint32_t)K)) return rc;
    } else {
        if (int rc = make_tmap_2d(&tb, b, (uint64_t)K, 128, (uint64_t)K, 64, 128)) return rc;
    }
    ProbeParams p{(const __nv_bfloat16*)a, out, ksteps, b_mn_major, a_from_regs, b_lbo, b_sbo, b_kstep_bytes};
    wgmma_probe_kernel<<<1, 288, 67 * 1024, (cudaStream_t)stream>>>(ta, tb, p);
    return check_launch("umma_probe");
}

// ------------------------------------------------------------------------------------------------
// library
// ------------------------------------------------------------------------------------------------
extern "C" int vcb_profile_begin(void) {
    Profiler& p = profiler();
    for (auto& r : p.recs) { p.pool.push_back(r.a); p.pool.push_back(r.b); }
    p.recs.clear();
    p.on = true;
    return 0;
}
namespace {
// categories beyond the caller's array fold into "other" (3), so the 4-entry form keeps summing every launch
int profile_collect(double* ms, long long* launches, int ncat, vcb_prof_record* recs, int64_t cap, int64_t* n_out) {
    if (!ms || !launches || ncat < 4 || ncat > PROF_NCAT) return set_error("profile_end: ncat must be in [4, %d]", (int)PROF_NCAT);
    Profiler& p = profiler();
    p.on = false;
    cudaError_t e = cudaDeviceSynchronize();
    if (e != cudaSuccess) return set_error("profile_end: %s", cudaGetErrorString(e));
    for (int i = 0; i < ncat; ++i) { ms[i] = 0.0; launches[i] = 0; }
    int64_t n = 0;
    for (auto& r : p.recs) {
        float t = 0.f;
        cudaEventElapsedTime(&t, r.a, r.b);
        const int c = r.cat < ncat ? r.cat : (int)PROF_OTHER;
        ms[c] += t;
        launches[c] += 1;
        if (recs && n < cap) {
            recs[n].category = r.cat;
            recs[n].ms = t;
            for (int k = 0; k < 4; ++k) recs[n].info[k] = r.info[k];
        }
        ++n;
        p.pool.push_back(r.a);
        p.pool.push_back(r.b);
    }
    if (n_out) *n_out = n;
    p.recs.clear();
    return 0;
}
}  // namespace
extern "C" int vcb_profile_end(double* ms, long long* launches) { return profile_collect(ms, launches, 4, nullptr, 0, nullptr); }
extern "C" int vcb_profile_end_ex(double* ms, long long* launches, int32_t ncat, vcb_prof_record* records, int64_t capacity,
                                  int64_t* n_records) {
    return profile_collect(ms, launches, ncat, records, capacity, n_records);
}
extern "C" int vcb_abi_version(void) { return VCB_ABI_VERSION; }
extern "C" const char* vcb_last_error(void) { return error_buf(); }
extern "C" long long vcb_launch_count(void) { return launch_counter().load(); }
extern "C" void vcb_reset_launch_count(void) { launch_counter().store(0); }
