// gemm_sm90.cuh -- persistent warp-specialised wgmma GEMM for sm_90a with fused epilogues.
//
//   D[M,N] = epilogue( A[M,K] (bf16, K-major) * W[N,K]^T (bf16, K-major), fp32 accumulate in registers )
//
// One CTA (or a cluster of two, cta_group 2) per SM, 384 threads:
//   warpgroup 0     TMA producer     one thread: global -> 128B-swizzled smem ring (mbarrier full/empty); registers handed over
//   warpgroups 1,2  consumers        rows [0,64) / [64,128) of the 128 x BLOCK_N tile: wgmma.mma_async from the ring, then the fused
//                                    epilogue straight from the accumulator registers while the producer prefetches the next tile
// cta_group 2: the two CTAs of a cluster work on a 256 x BLOCK_N tile; each loads its own 128 A rows and HALF of the B tile, which
// the TMA unit multicasts into both CTAs' rings -- B leaves L2 once per pair.
//
// Epilogues replace the reference's un-fused elementwise passes (SURVEY.md 2.2 / Appendix D) and keep the
// reference's bf16 rounding points under CUDA autocast (models/modules/layers.py:158-245).
#pragma once
#include "vcb_common.cuh"
#include "wgmma_sm90.cuh"

namespace vcb {

enum GemmEpilogue : int {
    EPI_BIAS = 0,       // out = bf16(acc + bias)
    EPI_BIAS_GELU = 1,  // out = bf16(gelu_tanh(bf16(acc + bias)))                         layers.py:143,154
    EPI_GATE_RES = 2,   // out = bf16(res + bf16(gate * bf16(acc + bias)))                  layers.py:190-195,245
    EPI_QKV = 3,        // q,k: bias -> QK-RMSNorm -> RoPE ; v: bias                        layers.py:165-174, math.py:112
    EPI_LINEAR1 = 4,    // cols < 3H as EPI_QKV into out ; cols >= 3H as EPI_BIAS_GELU into out2   layers.py:235-244
    EPI_BIAS_F32 = 5,   // out(fp32) = acc + bias   (VAE mid-block attention scores, autoencoder.py:47)
};
// EPI_GATE_RES with gate == nullptr is the plain residual epilogue out = bf16(res + bf16(acc + bias))
// (ResnetBlock / AttnBlock skip connections, autoencoder.py:52,82).

// A-operand addressing: a [batch, rows, K] matrix, or the 3x3 neighbourhood of an NHWC image (implicit GEMM, no im2col):
// k-block kb covers filter tap kb / (Cin/64) and channels 64*(kb % (Cin/64)); the tile's 128 rows are a 16 x 8 pixel
// patch loaded by ONE 4-D TMA box at the tap's (dx, dy) shift -- out-of-image pixels are zero-filled by the TMA unit,
// which is exactly the conv's zero padding.
enum GemmAMode : int { A_MATRIX = 0, A_CONV3X3 = 1 };
constexpr int kSpMaxRanks = 8;
constexpr int kConvTileW = 16, kConvTileH = 8;

struct GemmParams {
    int N, K;
    // A is a [batch, rows_per_batch, K] tensor (3-D TMA map; batch == 1 for a plain matrix).  M tiles never
    // straddle samples.  Row i of sample b is written to output row  b * out_batch_rows + out_row_offset + i,
    // which lets the txt / img streams read from and write to one joint [B, L, *] buffer without copies.
    int batch;
    int rows_per_batch;
    int out_batch_rows;
    int out_row_offset;
    // Tile raster.  0 (default): M-fastest -- the CTAs of a wave share few B (weight) tiles and cover all A rows.  1: N-fastest -- a
    // wave covers a band of A rows x ALL B tiles, A evict-first, B evict-last -- kept as an experiment switch.
    int n_fastest;
    const float* bias;           // [N] fp32 (may be null)
    // FP8 (e4m3) operands (kFp8 instantiations): acc is rescaled by a_scale[mapped output row] * w_scale[column] before the bias --
    // per-row activation scales written by the producing LayerNorm kernel, per-output-channel weight scales from packing time
    const float* a_scale;        // [rows of the joint buffer] fp32 (null = 1)
    const float* w_scale;        // [N] fp32 (null = 1)
    __nv_bfloat16* out;          // primary output
    long long ldo;               // elements
    int out_col_offset;
    // EPI_GATE_RES
    const __nv_bfloat16* gate;   // [B, gate_stride] bf16, column n
    long long gate_stride;
    const __nv_bfloat16* res;    // [rows, ld_res]; may alias out
    long long ld_res;
    // EPI_GATE_RES, optional: per-row partial sums of the bf16 residual stream this GEMM writes, one float2 (sum, sum of squares)
    // per 64 output columns at row_stats[orow * (N / 64) + column / 64] -- the statistics pass of the AdaLN LayerNorm that
    // follows (layers.py:191,195,234).  Every slot is written by exactly one thread: deterministic, no atomics.  Needs N % 64 == 0
    // and a tile whose column halves are multiples of 64 (BLOCK_N 128 or 256).
    float2* row_stats;
    // EPI_QKV / EPI_LINEAR1
    int hidden;                  // H (3H = end of the qkv columns); head_dim is 128
    const __nv_bfloat16* q_scale;  // [128] RMSNorm scale for q
    const __nv_bfloat16* k_scale;  // [128]
    const float2* rope;          // pair-major [64][rope_rows] (cos, sin); row index = the mapped output row
    long long rope_rows;
    __nv_bfloat16* out2;         // EPI_LINEAR1: gelu(mlp) destination
    long long ldo2;
    int out2_col_offset;
    // A_CONV3X3: OUTPUT height / width, input channels (K == 9 * conv_C); batch = images; rows_per_batch = H * W.
    // conv_stride 1 (pad 1 all round) or 2 (pad right/bottom only, autoencoder.py:91-95): for stride 2 the tensor map carries
    // elementStrides = 2, so one box still lands as a dense 16 x 8 pixel patch; coordinates are in input pixels.
    int conv_H, conv_W, conv_C, conv_stride;
    // Sequence-parallel head routing (EPI_QKV / EPI_LINEAR1, batch == 1; sp_world <= 1 = off).  Token rows are sharded over
    // sp_world ranks, heads over the same ranks for attention: the q/k/v columns of head h are stored straight into rank
    // h / (heads/W)'s peer-mapped qkv buffer [W * rows, 3 * hidden / W] over NVLink, at row sp_row_offset + output row.
    // The kernel's kSp instantiation writes each thread's 16-byte pieces through the peer-mapped pointers.
    int sp_world, sp_row_offset;
    __nv_bfloat16* sp_out[kSpMaxRanks];
    // Unmerged LoRA k-tail (bf16 operands): acc = A W^T + T B_lora^T, i.e. [A | T] [W | B_lora]^T.  After the ceil(K / 64)
    // k-blocks of (A, W) the producer loads ceil(lora_rank / 64) more from the T map (addressed like A: same rows_per_batch /
    // batch mapping) and the B_lora map (boxed like W, multicast like W under cta_group 2).  0 = no tail.
    int lora_rank;
    // output scale: the epilogue sees alpha * acc (0 = 1) -- the LoRA down-projection T = bf16(s * X A^T)
    float alpha;
};

// Stream-K tail (optional): the tiles of the partial last wave are cut along K into one equal contiguous range per CTA
// (pair), so no SM idles while a few CTAs finish whole tiles.  A split tile is produced by up to kSkMaxParts CTAs: the one
// holding the HEAD k range (kb0 == 0) finalises; the others dump fp32 partials to their workspace slot and raise a flag.
// A waiter only waits on CTAs with a larger index, whose contributing item is their FIRST item of the phase and waits on
// nothing: deadlock-free.  (Only the tail is split: with a fully contiguous stream-K
// over ALL tiles the CTAs of one wave no longer share B tiles.)
constexpr int kSkMaxParts = 8;
struct StreamKParams {
    float* ws;              // [gridDim.x][BLOCK_N / 2][256] fp32 partial accumulators (one slot per CTA, accumulator-register major)
    int* flags;             // [gridDim.x]
    int epoch;              // value that marks "partial of this launch is ready"
    int enabled;
};

struct WorkIter {
    // phase 1: the full waves with the plain strided schedule (CTA pairs of one wave share B tiles in L2);
    // phase 2 (stream-K only): the R = tiles % pairs tiles of the partial last wave are cut into equal contiguous
    // (tile, k-block) ranges, one per CTA pair.
    bool sk;
    int t, stride, full_tiles, num_tiles, num_kb;
    long long u, u1;
    __device__ __forceinline__ WorkIter(const StreamKParams& skp, int cluster_id, int num_clusters, int num_tiles_, int num_kb_)
        : sk(skp.enabled != 0), t(cluster_id), stride(num_clusters), num_tiles(num_tiles_), num_kb(num_kb_) {
        full_tiles = sk ? (num_tiles_ / num_clusters) * num_clusters : num_tiles_;
        const long long U = (long long)(num_tiles_ - full_tiles) * num_kb_;
        u = U * cluster_id / num_clusters;
        u1 = U * (cluster_id + 1) / num_clusters;
    }
    __device__ __forceinline__ bool next(int& tile, int& kb0, int& kb1) {
        if (t < full_tiles) {
            tile = t; kb0 = 0; kb1 = num_kb; t += stride;
            return true;
        }
        if (!sk || u >= u1) return false;
        const int lt = (int)(u / num_kb);
        tile = full_tiles + lt;
        kb0 = (int)(u - (long long)lt * num_kb);
        const long long rem = u1 - u;
        kb1 = rem < (long long)(num_kb - kb0) ? kb0 + (int)rem : num_kb;
        u += kb1 - kb0;
        return true;
    }
};


constexpr int kBlockM = 128;
constexpr int kBlockK = 64;
constexpr int kGemmThreads = 384;       // producer warpgroup + 2 consumer warpgroups
constexpr int kGemmConsumers = 256;

template <int BLOCK_N, int kCtaGroup>
struct GemmCfg {
    static constexpr int kBRows = BLOCK_N / kCtaGroup;           // B rows LOADED by one CTA (the whole tile lands in each CTA)
    static constexpr int kABytes = kBlockM * kBlockK * 2;        // 16 KB
    static constexpr int kBBytes = BLOCK_N * kBlockK * 2;
    static constexpr int kStageBytes = kABytes + kBBytes;
    static constexpr int kStages = (200 * 1024) / kStageBytes > 8 ? 8 : (200 * 1024) / kStageBytes;
    static constexpr int kSmemBytes = kStages * kStageBytes + 1024 /*align*/ + 256 /*barriers*/;
    static_assert(BLOCK_N % 32 == 0 && BLOCK_N <= 256, "BLOCK_N");
    static_assert((kBRows * kBlockK * 2) % 1024 == 0, "a CTA's share of the B tile keeps the 128-byte swizzle phase");
};

// ----------------------------------------------------------------------------------------------
// epilogue helpers
// ----------------------------------------------------------------------------------------------
// v = Linear output of 8 consecutive columns from n0: bf16 operands: bf16(acc + bias) (the reference's Linear returns bf16);
// fp8 (kRound false): fma(acc, sa * ws[n], bias) -- values are off the reference's grid already, the final store rounds once.
// sa: the row's activation scale; ws: per-column weight scales or null.  Columns >= N read no bias / scale.
template <bool kRound>
VCB_DEVICE void apply_bias8(float (&v)[8], const float* __restrict__ bias, const float* __restrict__ ws, float sa, int n0, int N) {
    float b[8], w[8];
    if (n0 + 8 <= N) {
        const float4 z = make_float4(0.f, 0.f, 0.f, 0.f), o = make_float4(1.f, 1.f, 1.f, 1.f);
        const float4 b0 = bias ? __ldg(reinterpret_cast<const float4*>(bias + n0)) : z, b1 = bias ? __ldg(reinterpret_cast<const float4*>(bias + n0) + 1) : z;
        const float4 w0 = ws ? __ldg(reinterpret_cast<const float4*>(ws + n0)) : o, w1 = ws ? __ldg(reinterpret_cast<const float4*>(ws + n0) + 1) : o;
        b[0] = b0.x; b[1] = b0.y; b[2] = b0.z; b[3] = b0.w; b[4] = b1.x; b[5] = b1.y; b[6] = b1.z; b[7] = b1.w;
        w[0] = w0.x; w[1] = w0.y; w[2] = w0.z; w[3] = w0.w; w[4] = w1.x; w[5] = w1.y; w[6] = w1.z; w[7] = w1.w;
    } else {
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            b[j] = (bias && n0 + j < N) ? __ldg(bias + n0 + j) : 0.f;
            w[j] = (ws && n0 + j < N) ? __ldg(ws + n0 + j) : 1.f;
        }
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        const float x = ws ? fmaf(v[j], sa * w[j], b[j]) : v[j] + b[j];
        v[j] = kRound ? bf16_round(x) : x;
    }
}

// ----------------------------------------------------------------------------------------------
// the kernel
// ----------------------------------------------------------------------------------------------
// kFp8: both operands are e4m3 bytes (K-major, 128 elements per 128-byte swizzle row); wgmma e4m3 x e4m3, K = 32 per instruction.
// A k-block is 128 bytes of K in either mode, so the pipeline (stage bytes, 4 MMAs of 32 bytes of K per k-block, descriptor
// advance) is unchanged; only the element count per k-block, the MMA kind and the epilogue's rescaling differ.
template <int BLOCK_N, int kCtaGroup, int kEpi, int kAMode = A_MATRIX, bool kSp = false, bool kFp8 = false>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_wgmma_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b, const GemmParams p,
                  const __grid_constant__ CUtensorMap tmap_a1, const __grid_constant__ CUtensorMap tmap_b1, const GemmParams p1,
                  const StreamKParams skp,
                  const __grid_constant__ CUtensorMap tmap_t, const __grid_constant__ CUtensorMap tmap_lb,
                  const __grid_constant__ CUtensorMap tmap_t1, const __grid_constant__ CUtensorMap tmap_lb1) {
    static_assert(!kSp || kEpi == EPI_QKV || kEpi == EPI_LINEAR1, "sequence-parallel routing lives in the head-structured epilogues");
    static_assert(!kFp8 || (kAMode == A_MATRIX && !kSp), "fp8 operands: plain matrices, single-GPU path");
    static_assert(kAMode == A_MATRIX || kCtaGroup == 1, "conv mode is single-CTA");
    static_assert((kEpi != EPI_QKV && kEpi != EPI_LINEAR1) || BLOCK_N % 128 == 0, "head-structured epilogue");
    constexpr int kBlockKEl = kFp8 ? 2 * kBlockK : kBlockK;          // elements of K per k-block (128 bytes either way)
    // Grouped launch: an optional second problem (p1.batch > 0) with the same N, K and epilogue but its own operands --
    // the txt stream of a DoubleStreamBlock rides in the img stream's launch and fills its partial last wave.
    using Cfg = GemmCfg<BLOCK_N, kCtaGroup>;
    constexpr int kStages = Cfg::kStages;
    constexpr int kAccRegs = BLOCK_N / 2;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint8_t* smem_a = smem;
    uint8_t* smem_b = smem + kStages * Cfg::kABytes;
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + kStages * Cfg::kStageBytes);   // [kStages]
    uint64_t* empty_bar = full_bar + kStages;                                                // [kStages]

    const uint32_t warp = warp_id_uniform();
    const uint32_t lane = lane_id();
    const uint32_t cta_rank = (kCtaGroup == 2) ? cluster_ctarank() : 0u;

    pdl_launch_dependents();
    if (warp == 0 && lane == 0) {
        tma_prefetch_desc(&tmap_a);
        tma_prefetch_desc(&tmap_b);
        if (p1.batch > 0) {
            tma_prefetch_desc(&tmap_a1);
            tma_prefetch_desc(&tmap_b1);
        }
        if (!kFp8 && kAMode == A_MATRIX && p.lora_rank > 0) {
            tma_prefetch_desc(&tmap_t);
            tma_prefetch_desc(&tmap_lb);
            if (p1.batch > 0) {
                tma_prefetch_desc(&tmap_t1);
                tma_prefetch_desc(&tmap_lb1);
            }
        }
        for (int s = 0; s < kStages; ++s) {
            mbar_init(&full_bar[s], 1);
            mbar_init(&empty_bar[s], 2 * kCtaGroup);      // one arrive per consumer warpgroup of every CTA the stage was sent to
        }
        fence_barrier_init();
    }
    if constexpr (kCtaGroup == 2) cluster_sync(); else __syncthreads();
    pdl_wait();                                     // everything above overlapped the previous kernel's tail

    const int tile_m = kBlockM * kCtaGroup;
    const int conv_tx = (kAMode == A_CONV3X3) ? (p.conv_W + kConvTileW - 1) / kConvTileW : 1;
    const int m_per_sample = (kAMode == A_CONV3X3) ? conv_tx * ((p.conv_H + kConvTileH - 1) / kConvTileH)
                                                   : (p.rows_per_batch + tile_m - 1) / tile_m;
    const int num_m = m_per_sample * p.batch;
    const int num_n = (p.N + BLOCK_N - 1) / BLOCK_N;
    const int tiles0 = num_m * num_n;
    const int m_per_sample1 = (p1.rows_per_batch + tile_m - 1) / tile_m;
    const int num_m1 = p1.batch > 0 ? m_per_sample1 * p1.batch : 0;
    const int num_tiles = tiles0 + num_m1 * num_n;
    // the LoRA k-tail adds its k-blocks behind the main ones, so the stream-K split and the grouped launch cover it unchanged
    // (both problems of a grouped launch share K and lora_rank)
    const int kb_main = (p.K + kBlockKEl - 1) / kBlockKEl;
    const int num_kb = kb_main + ((!kFp8 && kAMode == A_MATRIX) ? (p.lora_rank + kBlockK - 1) / kBlockK : 0);
    const int cluster_id = blockIdx.x / kCtaGroup;
    const int num_clusters = gridDim.x / kCtaGroup;

    if (warp < 4) {
        // ===================== TMA producer =====================
        setmaxnreg_dec<40>();
        if (warp == 0 && lane == 0) {
            int stage = 0;
            uint32_t phase = 0;
            WorkIter it(skp, cluster_id, num_clusters, num_tiles, num_kb);
            int t, kb0, kb1;
            while (it.next(t, kb0, kb1)) {
                const bool g1 = t >= tiles0;
                const int tt = g1 ? t - tiles0 : t, nm = g1 ? num_m1 : num_m, mps = g1 ? m_per_sample1 : m_per_sample;
                const CUtensorMap* ta = g1 ? &tmap_a1 : &tmap_a;
                const CUtensorMap* tb = g1 ? &tmap_b1 : &tmap_b;
                const int mt = p.n_fastest ? tt / num_n : tt % nm;
                const int bi = mt / mps;
                const int m0 = (mt % mps) * tile_m + (int)cta_rank * kBlockM;
                const int n0 = (p.n_fastest ? tt % num_n : tt / nm) * BLOCK_N + (int)cta_rank * Cfg::kBRows;
                const uint64_t hint_a = p.n_fastest ? kEvictFirst : kEvictNormal, hint_b = p.n_fastest ? kEvictLast : kEvictNormal;
                for (int kb = kb0; kb < kb1; ++kb) {
                    mbar_wait(&empty_bar[stage], phase ^ 1);
                    mbar_expect_tx(&full_bar[stage], Cfg::kStageBytes);
                    const bool tail = kb >= kb_main;       // LoRA k-tail: T in place of A, B_lora in place of W
                    const int kc = (tail ? kb - kb_main : kb) * kBlockKEl;
                    if constexpr (kAMode == A_CONV3X3) {
                        const int cpb = p.conv_C / kBlockK;
                        const int tap = kb / cpb, cb = kb - tap * cpb;
                        const int mi = mt % mps;
                        const int pad = p.conv_stride == 1 ? 1 : 0;
                        const int x0 = (mi % conv_tx) * kConvTileW * p.conv_stride + (tap % 3) - pad;
                        const int y0 = (mi / conv_tx) * kConvTileH * p.conv_stride + (tap / 3) - pad;
                        tma_load_4d(ta, &full_bar[stage], smem_a + stage * Cfg::kABytes, cb * kBlockK, x0, y0, bi, kEvictNormal);
                    } else {
                        tma_load_3d(tail ? (g1 ? &tmap_t1 : &tmap_t) : ta, &full_bar[stage], smem_a + stage * Cfg::kABytes, kc, m0, bi, hint_a);
                    }
                    tma_load_2d<kCtaGroup == 2>(tail ? (g1 ? &tmap_lb1 : &tmap_lb) : tb, &full_bar[stage],
                                                smem_b + stage * Cfg::kBBytes + (int)cta_rank * Cfg::kBRows * 128, kc, n0, hint_b, (uint16_t)3);
                    if (++stage == kStages) { stage = 0; phase ^= 1; }
                }
            }
        }
    } else {
        // ===================== consumer warpgroups: mainloop + epilogue =====================
        setmaxnreg_inc<232>();
        const int ctid = (int)threadIdx.x - 128;            // 0..255
        const int wg = ctid >> 7;                           // rows [64 wg, 64 wg + 64) of the CTA's 128
        const uint32_t q = lane & 3;
        const int frag_row = wg * 64 + (int)(warp & 3) * 16 + (int)(lane >> 2);     // + 8 h
        int stage = 0;
        uint32_t phase = 0;
        WorkIter it(skp, cluster_id, num_clusters, num_tiles, num_kb);
        int t, kb0, kb1;
        const int my_cta = cluster_id * kCtaGroup + (int)cta_rank;
        auto release = [&](int s) {                         // the warpgroup's wgmmas reading stage s have completed
            if ((warp & 3) == 0 && lane == 0) {
                if constexpr (kCtaGroup == 2) { mbar_arrive_cluster(&empty_bar[s], 0); mbar_arrive_cluster(&empty_bar[s], 1); }
                else mbar_arrive(&empty_bar[s]);
            }
        };
        float acc[kAccRegs];
        while (it.next(t, kb0, kb1)) {
            // ---------------- mainloop: one wgmma group (4 k steps) in flight behind the one being issued ----------------
            int prev = -1;
            for (int kb = kb0; kb < kb1; ++kb) {
                mbar_wait(&full_bar[stage], phase);
                const uint64_t a_desc = make_smem_desc(smem_u32(smem_a + stage * Cfg::kABytes + wg * 64 * 128), 16, 1024);
                const uint64_t b_desc = make_smem_desc(smem_u32(smem_b + stage * Cfg::kBBytes), 16, 1024);
                wgmma_fence();
#pragma unroll
                for (int k = 0; k < 4; ++k)     // 32 bytes of K per step inside the 128B swizzle span: +2 in the (addr >> 4) field
                    wgmma_ss<BLOCK_N, kFp8>(acc, a_desc + (uint64_t)(2 * k), b_desc + (uint64_t)(2 * k), (kb > kb0 || k != 0) ? 1u : 0u);
                wgmma_commit();
                if (prev >= 0) { wgmma_wait<1>(); release(prev); }
                prev = stage;
                if (++stage == kStages) { stage = 0; phase ^= 1; }
            }
            wgmma_wait<0>();
            release(prev);

            const bool g1 = t >= tiles0;
            const GemmParams& P = g1 ? p1 : p;
            const bool sk_contrib = kb0 > 0;                       // tail part of a split tile: dump partials, no epilogue
            const bool sk_final = !sk_contrib && kb1 < num_kb;     // head part: add the partners' partials, then epilogue
            if (sk_contrib) {
                // raw fp32 accumulators -> this CTA's workspace slot, register-major: consecutive threads write consecutive words
                float* slot = skp.ws + (long long)my_cta * kBlockM * BLOCK_N + ctid;
#pragma unroll
                for (int i = 0; i < kAccRegs; ++i) slot[i * kGemmConsumers] = acc[i];
                __threadfence();
                named_bar_sync(1, kGemmConsumers);                  // all consumer warps have written and fenced
                if (ctid == 0) st_release_gpu(skp.flags + my_cta, skp.epoch);
                continue;
            }
            if (sk_final) {
                // partners: the following CTA pairs (same rank) whose range starts inside this tile; each produced its part as
                // the FIRST item of its phase 2.  Fold their fp32 partials into my accumulators, then run the normal epilogue.
                const long long U = (long long)(num_tiles - it.full_tiles) * num_kb;
                const long long tile_end = (long long)(t - it.full_tiles + 1) * num_kb;
#pragma unroll 1
                for (int pc = cluster_id + 1; pc < num_clusters && U * pc / num_clusters < tile_end; ++pc) {
                    const int partner = pc * kCtaGroup + (int)cta_rank;
                    if (lane == 0) {
                        while (ld_acquire_gpu(skp.flags + partner) != skp.epoch) {
                        }
                    }
                    __syncwarp();
                    const float* part = skp.ws + (long long)partner * kBlockM * BLOCK_N + ctid;
#pragma unroll
                    for (int i = 0; i < kAccRegs; ++i) acc[i] += __ldcg(part + i * kGemmConsumers);
                }
            }
            if (P.alpha != 0.f && P.alpha != 1.f) {
#pragma unroll
                for (int i = 0; i < kAccRegs; ++i) acc[i] *= P.alpha;
            }

            // ---------------- epilogue: this thread's two rows (h = 0, 1: frag_row + 8 h) ----------------
            const int tt = g1 ? t - tiles0 : t, nm = g1 ? num_m1 : num_m, mps = g1 ? m_per_sample1 : m_per_sample;
            const int mt = p.n_fastest ? tt / num_n : tt % nm;
            const int b = mt / mps;
            const int n_tile0 = (p.n_fastest ? tt % num_n : tt / nm) * BLOCK_N;
            bool row_ok[2];
            long long orow[2];
            [[maybe_unused]] float sa[2];
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int row_in_tile = frag_row + 8 * h;
                int i;
                if constexpr (kAMode == A_CONV3X3) {
                    const int mi = mt % mps;
                    const int px = (mi % conv_tx) * kConvTileW + (row_in_tile % kConvTileW);
                    const int py = (mi / conv_tx) * kConvTileH + (row_in_tile / kConvTileW);
                    row_ok[h] = px < P.conv_W && py < P.conv_H;
                    i = py * P.conv_W + px;
                } else {
                    i = (mt % mps) * tile_m + (int)cta_rank * kBlockM + row_in_tile;
                    row_ok[h] = i < P.rows_per_batch;
                }
                orow[h] = (long long)b * P.out_batch_rows + P.out_row_offset + (row_ok[h] ? i : 0);
                sa[h] = (kFp8 && P.a_scale) ? __ldg(P.a_scale + orow[h]) : 1.0f;
            }
            [[maybe_unused]] const float* ws = kFp8 ? P.w_scale : nullptr;
            // intermediate roundings to the bf16 grid: the reference's autocast semantics; skipped for e4m3 operands (see apply_bias8)
            [[maybe_unused]] auto rnd = [](float x) { return kFp8 ? x : bf16_round(x); };

            if constexpr (kEpi == EPI_BIAS_F32) {
#pragma unroll
                for (int c = 0; c < BLOCK_N / 32; ++c) {
                    const int n0 = n_tile0 + c * 32 + 8 * (int)q;
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        float v[8];
                        frag_row8(acc, c, h, q, v);
                        if (row_ok[h] && n0 < P.N) {
                            float* dst = reinterpret_cast<float*>(P.out) + orow[h] * P.ldo + P.out_col_offset + n0;
#pragma unroll
                            for (int j = 0; j < 8; ++j) v[j] += (P.bias && n0 + j < P.N) ? __ldg(P.bias + n0 + j) : 0.f;
                            *reinterpret_cast<float4*>(dst) = make_float4(v[0], v[1], v[2], v[3]);
                            if (n0 + 4 < P.N) *reinterpret_cast<float4*>(dst + 4) = make_float4(v[4], v[5], v[6], v[7]);
                        }
                    }
                }
            } else if constexpr (kEpi == EPI_BIAS || kEpi == EPI_BIAS_GELU || kEpi == EPI_GATE_RES) {
                [[maybe_unused]] float st_sum[2] = {0.f, 0.f}, st_sq[2] = {0.f, 0.f};
#pragma unroll
                for (int c = 0; c < BLOCK_N / 32; ++c) {
                    const int n0 = n_tile0 + c * 32 + 8 * (int)q;
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        float v[8];
                        frag_row8(acc, c, h, q, v);
                        const bool in = row_ok[h] && n0 < P.N;
                        if (in) {
                            apply_bias8<!kFp8>(v, P.bias, ws, sa[h], n0, P.N);
                            if constexpr (kEpi == EPI_BIAS_GELU) {
#pragma unroll
                                for (int j = 0; j < 8; ++j) v[j] = kFp8 ? gelu_tanh_fast(v[j]) : gelu_tanh(v[j]);
                            }
                            if constexpr (kEpi == EPI_GATE_RES) {
                                const uint32_t one2 = 0x3F803F80u;          // bf16 (1.0, 1.0)
                                const uint4 gu = P.gate ? __ldg(reinterpret_cast<const uint4*>(P.gate + (long long)b * P.gate_stride + n0))
                                                        : make_uint4(one2, one2, one2, one2);
                                const uint4 ru = *reinterpret_cast<const uint4*>(P.res + orow[h] * P.ld_res + n0);
                                const uint32_t gw[4] = {gu.x, gu.y, gu.z, gu.w}, rw[4] = {ru.x, ru.y, ru.z, ru.w};
#pragma unroll
                                for (int e = 0; e < 4; ++e) {
                                    const float2 gf = unpack_bf16x2(gw[e]), rf = unpack_bf16x2(rw[e]);
                                    v[2 * e] = rf.x + rnd(gf.x * v[2 * e]);
                                    v[2 * e + 1] = rf.y + rnd(gf.y * v[2 * e + 1]);
                                }
                            }
                            store_bf16x8(P.out + orow[h] * P.ldo + P.out_col_offset + n0, v);
                        }
                        if constexpr (kEpi == EPI_GATE_RES && kAMode == A_MATRIX && BLOCK_N % 64 == 0) {
                            if (P.row_stats != nullptr) {           // uniform: every lane takes part in the quad reduction
                                // statistics of the values as STORED (bf16): the LayerNorm reads the stream back in bf16
#pragma unroll
                                for (int j = 0; j < 8; ++j) {
                                    const float xr = in ? bf16_round(v[j]) : 0.f;
                                    st_sum[h] += xr;
                                    st_sq[h] = fmaf(xr, xr, st_sq[h]);
                                }
                                if (c & 1) {
                                    const float s = quad_sum(st_sum[h]), s2 = quad_sum(st_sq[h]);
                                    if (q == 0 && row_ok[h] && n_tile0 + c * 32 < P.N)
                                        P.row_stats[orow[h] * (long long)(P.N >> 6) + ((n_tile0 + c * 32) >> 6)] = make_float2(s, s2);
                                    st_sum[h] = 0.f; st_sq[h] = 0.f;
                                }
                            }
                        }
                    }
                }
            } else {
                // EPI_QKV / EPI_LINEAR1: 128-column groups (one head each)
#pragma unroll
                for (int hg = 0; hg < BLOCK_N / 128; ++hg) {
                    const int ng = n_tile0 + hg * 128;           // first column of this 128-group
                    if (ng >= P.N) continue;
                    const int region = ng / P.hidden;            // 0 q, 1 k, 2 v, >= 3 mlp (LINEAR1)
                    // destination of this head's 128 q / k / v columns: the local qkv buffer, or (sequence-parallel) the
                    // qkv buffer of the rank that owns the head, through its peer-mapped pointer
                    __nv_bfloat16* qkv_dst[2];
#pragma unroll
                    for (int h = 0; h < 2; ++h) qkv_dst[h] = P.out + orow[h] * P.ldo + P.out_col_offset + ng;
                    if constexpr (kSp) {
                        if (region < 3) {
                            const int hw = P.hidden / P.sp_world;    // q (or k, v) columns per rank
                            const int cin = ng - region * P.hidden;
                            const int owner = cin / hw;
#pragma unroll
                            for (int h = 0; h < 2; ++h)
                                qkv_dst[h] = P.sp_out[owner] + ((long long)P.sp_row_offset + orow[h]) * (3LL * hw) + region * hw + (cin - owner * hw);
                        }
                    }
                    if (region >= 2) {
#pragma unroll
                        for (int c = 0; c < 4; ++c) {
                            const int n0 = ng + c * 32 + 8 * (int)q;
#pragma unroll
                            for (int h = 0; h < 2; ++h) {
                                float v[8];
                                frag_row8(acc, hg * 4 + c, h, q, v);
                                if (!row_ok[h] || n0 >= P.N) continue;
                                apply_bias8<!kFp8>(v, P.bias, ws, sa[h], n0, P.N);
                                if (kEpi == EPI_LINEAR1 && region >= 3) {
#pragma unroll
                                    for (int j = 0; j < 8; ++j) v[j] = kFp8 ? gelu_tanh_fast(v[j]) : gelu_tanh(v[j]);
                                    store_bf16x8(P.out2 + orow[h] * P.ldo2 + P.out2_col_offset + (n0 - 3 * P.hidden), v);
                                } else {
                                    store_bf16x8(qkv_dst[h] + c * 32 + 8 * (int)q, v);
                                }
                            }
                        }
                    } else {
                        const __nv_bfloat16* sc = region == 0 ? P.q_scale : P.k_scale;
                        // pass 1: sum of squares of the (bf16-rounded) projection over the head (RMSNorm, layers.py:68-72), on the
                        // accumulator's own column pairs 8 j + 2 q, then across the quad
                        float ss[2] = {0.f, 0.f};
#pragma unroll
                        for (int j = 0; j < 16; ++j) {
                            const int n = ng + 8 * j + 2 * (int)q;
                            const float2 bj = P.bias ? __ldg(reinterpret_cast<const float2*>(P.bias + n)) : make_float2(0.f, 0.f);
                            const float2 wj = ws ? __ldg(reinterpret_cast<const float2*>(ws + n)) : make_float2(1.f, 1.f);
#pragma unroll
                            for (int h = 0; h < 2; ++h) {
                                const float a0 = acc[(hg * 16 + j) * 4 + 2 * h], a1 = acc[(hg * 16 + j) * 4 + 2 * h + 1];
                                const float x0 = ws ? fmaf(a0, sa[h] * wj.x, bj.x) : rnd(a0 + bj.x);
                                const float x1 = ws ? fmaf(a1, sa[h] * wj.y, bj.y) : rnd(a1 + bj.y);
                                ss[h] = fmaf(x0, x0, fmaf(x1, x1, ss[h]));
                            }
                        }
                        float rrms[2];
#pragma unroll
                        for (int h = 0; h < 2; ++h) rrms[h] = rsqrtf(quad_sum(ss[h]) * (1.0f / 128.0f) + 1e-6f);
                        // pass 2: normalise, scale, rotate, store.  The rope table is pair-major [64][rope_rows] (cos, sin).
#pragma unroll
                        for (int c = 0; c < 4; ++c) {
                            const int d0 = c * 32 + 8 * (int)q;          // my 8 columns inside the head
                            const uint4 su = __ldg(reinterpret_cast<const uint4*>(sc + d0));
                            const uint32_t sw[4] = {su.x, su.y, su.z, su.w};
#pragma unroll
                            for (int h = 0; h < 2; ++h) {
                                float v[8];
                                frag_row8(acc, hg * 4 + c, h, q, v);
                                if (!row_ok[h]) continue;
                                apply_bias8<!kFp8>(v, P.bias, ws, sa[h], ng + d0, P.N);
                                const float2* rp = P.rope + orow[h] + (long long)(d0 >> 1) * P.rope_rows;
#pragma unroll
                                for (int e = 0; e < 4; ++e) {
                                    const float2 s2 = unpack_bf16x2(sw[e]);
                                    const float x0 = rnd(rnd(v[2 * e] * rrms[h]) * s2.x);
                                    const float x1 = rnd(rnd(v[2 * e + 1] * rrms[h]) * s2.y);
                                    const float2 cs = __ldg(rp + (long long)e * P.rope_rows);
                                    // math.py:112-117: two fp32 products, one fp32 add (no contraction)
                                    v[2 * e] = __fadd_rn(__fmul_rn(cs.x, x0), __fmul_rn(-cs.y, x1));
                                    v[2 * e + 1] = __fadd_rn(__fmul_rn(cs.y, x0), __fmul_rn(cs.x, x1));
                                }
                                store_bf16x8(qkv_dst[h] + d0, v);
                            }
                        }
                    }
                }
            }
        }
    }

    // a CTA of a pair must not exit while its peer can still multicast into it or arrive on its barriers
    if constexpr (kCtaGroup == 2) cluster_sync();
}

}  // namespace vcb
