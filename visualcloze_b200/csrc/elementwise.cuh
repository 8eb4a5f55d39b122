// elementwise.cuh -- HBM-bound helpers of the FLUX-DiT step (coalesced 16-byte accesses, fp32 math).
#pragma once
#include "vcb_common.cuh"

namespace vcb {

// ------------------------------------------------------------------------------------------------
// AdaLN: y = bf16( bf16(1 + scale) * LayerNorm(x) + shift ), LayerNorm without affine, eps 1e-6, fp32 stats.
// Replaces F.layer_norm + two elementwise passes + the autocast cast (layers.py:163-164,191,195,234,257).
// One warp per row; the row stays in registers between the statistics and the modulation.
// Algorithmic bytes: read + write of [rows, H] bf16 = 4*rows*H bytes.
// ------------------------------------------------------------------------------------------------
constexpr int kLnMaxChunks = 16;      // 16 * 256 = up to H = 4096 per row
constexpr int kLnWarps = 8;           // rows per block iteration

// One warp per row, 8 rows per block.  The block's modulation vectors (shift, 1 + scale) are staged once in shared
// memory as bf16 pairs; a row is read once (16-byte loads, kept packed in registers), statistics are taken in one pass
// (sum and sum of squares in fp32), and the modulated row is written once.
// One launch may carry two problems (the img and txt streams of a DoubleStreamBlock, layers.py:163 / 170): blocks
// [0, p0.blocks) work on p0, the rest on p1.
struct LnProblem {
    const __nv_bfloat16* x; __nv_bfloat16* y;
    const __nv_bfloat16* shift; const __nv_bfloat16* scale;
    int rows, rows_per_batch, blocks;
};
// kChunks = H / 256 at compile time: the row lives in kChunks uint4 registers per lane (12 for H = 3072), which keeps the kernel
// at 3 blocks per SM; the generic instantiation (kLnMaxChunks) serves every other hidden size.
template <int kChunks, int kMinBlocks>
__global__ void __launch_bounds__(kLnWarps * 32, kMinBlocks)
ln_modulate_kernel(const LnProblem p0, const LnProblem p1, long long ldx, long long ldy, long long mod_stride, int H, int batch_rows) {
    extern __shared__ uint4 ln_smem[];                 // [2][H / 8] : shift, scale of sample b0
    pdl_launch_dependents();
    pdl_wait();
    const bool second = (int)blockIdx.x >= p0.blocks;
    const LnProblem& P = second ? p1 : p0;
    const __nv_bfloat16* __restrict__ x = P.x;
    __nv_bfloat16* __restrict__ y = P.y;
    const __nv_bfloat16* __restrict__ shift = P.shift;
    const __nv_bfloat16* __restrict__ scale = P.scale;
    const int rows = P.rows, rows_per_batch = P.rows_per_batch;
    const int row0 = ((int)blockIdx.x - (second ? p0.blocks : 0)) * kLnWarps;
    const int b0 = row0 / rows_per_batch;
    const int nvec = H >> 3;
    for (int i = threadIdx.x; i < 2 * nvec; i += blockDim.x) {
        const __nv_bfloat16* src = (i < nvec ? shift : scale) + (long long)b0 * mod_stride;
        ln_smem[i] = __ldg(reinterpret_cast<const uint4*>(src) + (i < nvec ? i : i - nvec));
    }
    const int row = row0 + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    const int nchunks = H >> 8;                    // H % 256 == 0
    const bool active = row < rows;
    const int b = active ? row / rows_per_batch : b0;
    // logical row (b, i) lives at physical row b * batch_rows + i of x and y (a stream inside a joint [B, L, H] buffer)
    const long long prow = (long long)b * batch_rows + (row - b * rows_per_batch);
    uint4 v[kChunks];
    float sum = 0.f, sq = 0.f;
    if (active) {
        const __nv_bfloat16* xr = x + prow * ldx;
#pragma unroll
        for (int c = 0; c < kChunks; ++c)
            if (c < nchunks) v[c] = *reinterpret_cast<const uint4*>(xr + c * 256 + lane * 8);
#pragma unroll
        for (int c = 0; c < kChunks; ++c)
            if (c < nchunks) {
                const uint32_t w[4] = {v[c].x, v[c].y, v[c].z, v[c].w};
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    float2 f = unpack_bf16x2(w[e]);
                    sum += f.x + f.y;
                    sq = fmaf(f.x, f.x, fmaf(f.y, f.y, sq));
                }
            }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        sum += __shfl_xor_sync(0xffffffffu, sum, o);
        sq += __shfl_xor_sync(0xffffffffu, sq, o);
    }
    __syncthreads();                                // modulation vectors staged
    if (!active) return;
    const float mean = sum / (float)H;
    const float var = fmaxf(sq / (float)H - mean * mean, 0.f);
    const float rstd = rsqrtf(var + 1e-6f);
    const bool staged = (b == b0);
    const uint4* sh_g = reinterpret_cast<const uint4*>(shift + (long long)b * mod_stride);
    const uint4* sc_g = reinterpret_cast<const uint4*>(scale + (long long)b * mod_stride);
    __nv_bfloat16* yr = y + prow * ldy;
#pragma unroll
    for (int c = 0; c < kChunks; ++c)
        if (c < nchunks) {
            const int vi = c * 32 + lane;
            const uint4 hu = staged ? ln_smem[vi] : __ldg(sh_g + vi);
            const uint4 su = staged ? ln_smem[nvec + vi] : __ldg(sc_g + vi);
            const uint32_t xw[4] = {v[c].x, v[c].y, v[c].z, v[c].w};
            const uint32_t sw[4] = {su.x, su.y, su.z, su.w};
            const uint32_t hw[4] = {hu.x, hu.y, hu.z, hu.w};
            uint32_t ow[4];
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                float2 xf = unpack_bf16x2(xw[e]);
                float2 s2 = unpack_bf16x2(sw[e]);
                float2 h2 = unpack_bf16x2(hw[e]);
                // `1 + scale` is a bf16 op in the reference; the product and sum are fp32 (LayerNorm returns fp32)
                float a0 = bf16_round(1.0f + s2.x), a1 = bf16_round(1.0f + s2.y);
                float n0 = (xf.x - mean) * rstd, n1 = (xf.y - mean) * rstd;
                ow[e] = pack_bf16x2(__fadd_rn(__fmul_rn(a0, n0), h2.x), __fadd_rn(__fmul_rn(a1, n1), h2.y));
            }
            *reinterpret_cast<uint4*>(yr + c * 256 + lane * 8) = make_uint4(ow[0], ow[1], ow[2], ow[3]);
        }
}

// Two-pass variant (default): the row is NOT kept in registers between the statistics and the modulation -- pass 2 re-reads
// it (L1 / L2 hits: the warp has just touched those lines).  That frees ~48 registers per thread, so 5 blocks x 8 warps fit an
// SM and 148 x 40 = 5920 warps are resident: every row of a cfg-B sequence (3968) is in flight in ONE round.  The one-pass
// kernel above holds 3 blocks per SM = 3552 warps: 3968 rows took two rounds of which the second was 12 % full -- that, not
// bandwidth, was its 25 us (ncu: 13.7 % DRAM throughput).  Same arithmetic in the same order: results are bit-identical.
__global__ void __launch_bounds__(kLnWarps * 32, 5)
ln_modulate2_kernel(const LnProblem p0, const LnProblem p1, long long ldx, long long ldy, long long mod_stride, int H, int batch_rows) {
    // [2][H] fp32: bf16(1 + scale) and shift of sample b0, converted ONCE per block -- the per-element work of pass 2 drops from
    // ~25 to ~13 instructions per bf16 pair (the kernel was as much issue-bound as latency-bound: 12 M elements x 12 instructions)
    extern __shared__ float4 ln_smem4[];
    pdl_launch_dependents();
    pdl_wait();
    const bool second = (int)blockIdx.x >= p0.blocks;
    const LnProblem& P = second ? p1 : p0;
    const int rows = P.rows, rows_per_batch = P.rows_per_batch;
    const int row0 = ((int)blockIdx.x - (second ? p0.blocks : 0)) * kLnWarps;
    const int b0 = row0 / rows_per_batch;
    const int nvec = H >> 3;                       // 8-element groups per row
    const int row = row0 + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    const int nchunks = H >> 8;                    // H % 256 == 0
    const bool active = row < rows;
    const int b = active ? row / rows_per_batch : b0;
    const long long prow = (long long)b * batch_rows + (row - b * rows_per_batch);
    const uint4* xr = reinterpret_cast<const uint4*>(P.x + prow * ldx) + lane;
    // pass 1: statistics, four 16-byte loads in flight per lane (48 warps per SM keep ~100 KB in flight)
    float sum = 0.f, sq = 0.f;
    if (active) {
#pragma unroll 4
        for (int c = 0; c < nchunks; ++c) {
            const uint4 v = xr[c * 32];
            const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                float2 f = unpack_bf16x2(w[e]);
                sum += f.x + f.y;
                sq = fmaf(f.x, f.x, fmaf(f.y, f.y, sq));
            }
        }
    }
    // group i (8 elements) of the modulation row -> four float4 planes (consecutive lanes read consecutive float4: no bank conflicts):
    // a = bf16(1 + scale) (a bf16 op in the reference) elements 0-3 at [i], 4-7 at [nvec + i]; shift at [2 nvec + i], [3 nvec + i]
    for (int i = threadIdx.x; i < nvec; i += blockDim.x) {
        const uint4 su = __ldg(reinterpret_cast<const uint4*>(P.scale + (long long)b0 * mod_stride) + i);
        const uint4 hu = __ldg(reinterpret_cast<const uint4*>(P.shift + (long long)b0 * mod_stride) + i);
        const float2 s0 = unpack_bf16x2(su.x), s1 = unpack_bf16x2(su.y), s2 = unpack_bf16x2(su.z), s3 = unpack_bf16x2(su.w);
        const float2 h0 = unpack_bf16x2(hu.x), h1 = unpack_bf16x2(hu.y), h2 = unpack_bf16x2(hu.z), h3 = unpack_bf16x2(hu.w);
        ln_smem4[i] = make_float4(bf16_round(1.0f + s0.x), bf16_round(1.0f + s0.y), bf16_round(1.0f + s1.x), bf16_round(1.0f + s1.y));
        ln_smem4[nvec + i] = make_float4(bf16_round(1.0f + s2.x), bf16_round(1.0f + s2.y), bf16_round(1.0f + s3.x), bf16_round(1.0f + s3.y));
        ln_smem4[2 * nvec + i] = make_float4(h0.x, h0.y, h1.x, h1.y);
        ln_smem4[3 * nvec + i] = make_float4(h2.x, h2.y, h3.x, h3.y);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        sum += __shfl_xor_sync(0xffffffffu, sum, o);
        sq += __shfl_xor_sync(0xffffffffu, sq, o);
    }
    __syncthreads();                                // modulation vectors staged
    if (!active) return;
    const float mean = sum / (float)H;
    const float var = fmaxf(sq / (float)H - mean * mean, 0.f);
    const float rstd = rsqrtf(var + 1e-6f);
    const bool staged = (b == b0);
    const uint4* sh_g = reinterpret_cast<const uint4*>(P.shift + (long long)b * mod_stride);
    const uint4* sc_g = reinterpret_cast<const uint4*>(P.scale + (long long)b * mod_stride);
    uint4* yr = reinterpret_cast<uint4*>(P.y + prow * ldy) + lane;
    // pass 2: re-read, modulate, write
#pragma unroll 2
    for (int c = 0; c < nchunks; ++c) {
        const int vi = c * 32 + lane;
        const uint4 xv = xr[c * 32];
        float4 a0, a1, h0, h1;
        if (staged) {
            a0 = ln_smem4[vi]; a1 = ln_smem4[nvec + vi]; h0 = ln_smem4[2 * nvec + vi]; h1 = ln_smem4[3 * nvec + vi];
        } else {                                    // a block straddling two samples: this row's vectors straight from global
            const uint4 su = __ldg(sc_g + vi), hu = __ldg(sh_g + vi);
            const float2 s0 = unpack_bf16x2(su.x), s1 = unpack_bf16x2(su.y), s2 = unpack_bf16x2(su.z), s3 = unpack_bf16x2(su.w);
            const float2 g0 = unpack_bf16x2(hu.x), g1 = unpack_bf16x2(hu.y), g2 = unpack_bf16x2(hu.z), g3 = unpack_bf16x2(hu.w);
            a0 = make_float4(bf16_round(1.0f + s0.x), bf16_round(1.0f + s0.y), bf16_round(1.0f + s1.x), bf16_round(1.0f + s1.y));
            a1 = make_float4(bf16_round(1.0f + s2.x), bf16_round(1.0f + s2.y), bf16_round(1.0f + s3.x), bf16_round(1.0f + s3.y));
            h0 = make_float4(g0.x, g0.y, g1.x, g1.y);
            h1 = make_float4(g2.x, g2.y, g3.x, g3.y);
        }
        // the product and the sum are separate fp32 operations (LayerNorm returns fp32, then (1 + scale) * ln + shift)
        auto mod2 = [&](uint32_t xw, float ax, float ay, float hx, float hy) {
            const float2 xf = unpack_bf16x2(xw);
            const float n0 = (xf.x - mean) * rstd, n1 = (xf.y - mean) * rstd;
            return pack_bf16x2(__fadd_rn(__fmul_rn(ax, n0), hx), __fadd_rn(__fmul_rn(ay, n1), hy));
        };
        uint32_t ow[4];
        ow[0] = mod2(xv.x, a0.x, a0.y, h0.x, h0.y);
        ow[1] = mod2(xv.y, a0.z, a0.w, h0.z, h0.w);
        ow[2] = mod2(xv.z, a1.x, a1.y, h1.x, h1.y);
        ow[3] = mod2(xv.w, a1.z, a1.w, h1.z, h1.w);
        yr[c * 32] = make_uint4(ow[0], ow[1], ow[2], ow[3]);
    }
}

// Statistics-from-the-producer variant: the GATE_RES epilogue of the GEMM that wrote the residual stream also left, per row, one
// (sum, sum of squares) pair per 64 columns (gemm_sm90.cuh, row_stats).  The LayerNorm then needs no pass over the row for its
// statistics: a warp adds the row's n_slots pairs in a fixed order (deterministic), and streams the row ONCE.
struct LnStatsProblem {
    const __nv_bfloat16* x; __nv_bfloat16* y;
    const __nv_bfloat16* shift; const __nv_bfloat16* scale;
    const float2* stats;                            // [rows of this problem][n_slots], indexed by the physical row like x
    int rows, rows_per_batch, blocks;
};
// 4 blocks x 8 warps per SM = 4736 resident warps >= the 3968 rows of a cfg-B sequence: still one round, and 64 registers let a
// lane keep six 16-byte loads in flight -- the kernel is latency-bound (ncu: 16 us for 24 MB, one dependent chain per warp), so the
// row is covered by two batches of loads instead of four.
__global__ void __launch_bounds__(kLnWarps * 32, 4)
ln_modulate_stats_kernel(const LnStatsProblem p0, const LnStatsProblem p1, long long ldx, long long ldy, long long mod_stride, int H,
                         int batch_rows, int n_slots) {
    extern __shared__ float4 ln_smem4[];
    pdl_launch_dependents();
    pdl_wait();
    const bool second = (int)blockIdx.x >= p0.blocks;
    const LnStatsProblem& P = second ? p1 : p0;
    const int rows = P.rows, rows_per_batch = P.rows_per_batch;
    const int row0 = ((int)blockIdx.x - (second ? p0.blocks : 0)) * kLnWarps;
    const int b0 = row0 / rows_per_batch;
    const int nvec = H >> 3;
    const int row = row0 + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    const int nchunks = H >> 8;
    const bool active = row < rows;
    const int b = active ? row / rows_per_batch : b0;
    const long long prow = (long long)b * batch_rows + (row - b * rows_per_batch);
    float sum = 0.f, sq = 0.f;
    if (active) {
        const float2* st = P.stats + prow * n_slots;
        for (int i = lane; i < n_slots; i += 32) {
            const float2 v = __ldg(st + i);
            sum += v.x;
            sq += v.y;
        }
    }
    for (int i = threadIdx.x; i < nvec; i += blockDim.x) {
        const uint4 su = __ldg(reinterpret_cast<const uint4*>(P.scale + (long long)b0 * mod_stride) + i);
        const uint4 hu = __ldg(reinterpret_cast<const uint4*>(P.shift + (long long)b0 * mod_stride) + i);
        const float2 s0 = unpack_bf16x2(su.x), s1 = unpack_bf16x2(su.y), s2 = unpack_bf16x2(su.z), s3 = unpack_bf16x2(su.w);
        const float2 h0 = unpack_bf16x2(hu.x), h1 = unpack_bf16x2(hu.y), h2 = unpack_bf16x2(hu.z), h3 = unpack_bf16x2(hu.w);
        ln_smem4[i] = make_float4(bf16_round(1.0f + s0.x), bf16_round(1.0f + s0.y), bf16_round(1.0f + s1.x), bf16_round(1.0f + s1.y));
        ln_smem4[nvec + i] = make_float4(bf16_round(1.0f + s2.x), bf16_round(1.0f + s2.y), bf16_round(1.0f + s3.x), bf16_round(1.0f + s3.y));
        ln_smem4[2 * nvec + i] = make_float4(h0.x, h0.y, h1.x, h1.y);
        ln_smem4[3 * nvec + i] = make_float4(h2.x, h2.y, h3.x, h3.y);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        sum += __shfl_xor_sync(0xffffffffu, sum, o);
        sq += __shfl_xor_sync(0xffffffffu, sq, o);
    }
    __syncthreads();
    if (!active) return;
    const float mean = sum / (float)H;
    const float var = fmaxf(sq / (float)H - mean * mean, 0.f);
    const float rstd = rsqrtf(var + 1e-6f);
    const bool staged = (b == b0);
    const uint4* sh_g = reinterpret_cast<const uint4*>(P.shift + (long long)b * mod_stride);
    const uint4* sc_g = reinterpret_cast<const uint4*>(P.scale + (long long)b * mod_stride);
    const uint4* xr = reinterpret_cast<const uint4*>(P.x + prow * ldx) + lane;
    uint4* yr = reinterpret_cast<uint4*>(P.y + prow * ldy) + lane;
#pragma unroll 6
    for (int c = 0; c < nchunks; ++c) {
        const int vi = c * 32 + lane;
        const uint4 xv = xr[c * 32];
        float4 a0, a1, h0, h1;
        if (staged) {
            a0 = ln_smem4[vi]; a1 = ln_smem4[nvec + vi]; h0 = ln_smem4[2 * nvec + vi]; h1 = ln_smem4[3 * nvec + vi];
        } else {
            const uint4 su = __ldg(sc_g + vi), hu = __ldg(sh_g + vi);
            const float2 s0 = unpack_bf16x2(su.x), s1 = unpack_bf16x2(su.y), s2 = unpack_bf16x2(su.z), s3 = unpack_bf16x2(su.w);
            const float2 g0 = unpack_bf16x2(hu.x), g1 = unpack_bf16x2(hu.y), g2 = unpack_bf16x2(hu.z), g3 = unpack_bf16x2(hu.w);
            a0 = make_float4(bf16_round(1.0f + s0.x), bf16_round(1.0f + s0.y), bf16_round(1.0f + s1.x), bf16_round(1.0f + s1.y));
            a1 = make_float4(bf16_round(1.0f + s2.x), bf16_round(1.0f + s2.y), bf16_round(1.0f + s3.x), bf16_round(1.0f + s3.y));
            h0 = make_float4(g0.x, g0.y, g1.x, g1.y);
            h1 = make_float4(g2.x, g2.y, g3.x, g3.y);
        }
        auto mod2 = [&](uint32_t xw, float ax, float ay, float hx, float hy) {
            const float2 xf = unpack_bf16x2(xw);
            const float n0 = (xf.x - mean) * rstd, n1 = (xf.y - mean) * rstd;
            return pack_bf16x2(__fadd_rn(__fmul_rn(ax, n0), hx), __fadd_rn(__fmul_rn(ay, n1), hy));
        };
        uint32_t ow[4];
        ow[0] = mod2(xv.x, a0.x, a0.y, h0.x, h0.y);
        ow[1] = mod2(xv.y, a0.z, a0.w, h0.z, h0.w);
        ow[2] = mod2(xv.z, a1.x, a1.y, h1.x, h1.y);
        ow[3] = mod2(xv.w, a1.z, a1.w, h1.z, h1.w);
        yr[c * 32] = make_uint4(ow[0], ow[1], ow[2], ow[3]);
    }
}

// FP8 variant (opt-in fp8 projections): same statistics and modulation, but the row leaves as e4m3 bytes with ONE fp32 scale per
// row: s = max|y| / 448, y8 = e4m3(y / s).  The fp8 GEMM multiplies its accumulator by s (a_scale) again.  The modulated row is
// kept in registers between the amax and the quantisation (one warp per row, 3 blocks per SM like the one-pass bf16 kernel).
VCB_DEVICE uint32_t pack_e4m3x4(float a, float b, float c, float d) {
    uint16_t lo, hi;
    asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(lo) : "f"(b), "f"(a));      // first source -> upper byte
    asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(hi) : "f"(d), "f"(c));
    return (uint32_t)lo | ((uint32_t)hi << 16);
}
struct LnFp8Problem {
    const __nv_bfloat16* x; uint8_t* y8; float* row_scale;        // row_scale is indexed by the PHYSICAL row of the joint buffer
    const __nv_bfloat16* shift; const __nv_bfloat16* scale;
    int rows, rows_per_batch, blocks;
};
template <int kChunks>
__global__ void __launch_bounds__(kLnWarps * 32, 3)
ln_modulate_fp8_kernel(const LnFp8Problem p0, const LnFp8Problem p1, long long ldx, long long ldy, long long mod_stride, int H,
                       int batch_rows) {
    extern __shared__ uint4 ln_smem[];                 // [2][H / 8] : shift, scale of sample b0
    pdl_launch_dependents();
    pdl_wait();
    const bool second = (int)blockIdx.x >= p0.blocks;
    const LnFp8Problem& P = second ? p1 : p0;
    const int rows = P.rows, rows_per_batch = P.rows_per_batch;
    const int row0 = ((int)blockIdx.x - (second ? p0.blocks : 0)) * kLnWarps;
    const int b0 = row0 / rows_per_batch;
    const int nvec = H >> 3;
    for (int i = threadIdx.x; i < 2 * nvec; i += blockDim.x) {
        const __nv_bfloat16* src = (i < nvec ? P.shift : P.scale) + (long long)b0 * mod_stride;
        ln_smem[i] = __ldg(reinterpret_cast<const uint4*>(src) + (i < nvec ? i : i - nvec));
    }
    const int row = row0 + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    const int nchunks = H >> 8;
    const bool active = row < rows;
    const int b = active ? row / rows_per_batch : b0;
    const long long prow = (long long)b * batch_rows + (row - b * rows_per_batch);
    uint4 v[kChunks];
    float sum = 0.f, sq = 0.f;
    if (active) {
        const __nv_bfloat16* xr = P.x + prow * ldx;
#pragma unroll
        for (int c = 0; c < kChunks; ++c)
            if (c < nchunks) v[c] = *reinterpret_cast<const uint4*>(xr + c * 256 + lane * 8);
#pragma unroll
        for (int c = 0; c < kChunks; ++c)
            if (c < nchunks) {
                const uint32_t w[4] = {v[c].x, v[c].y, v[c].z, v[c].w};
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    float2 f = unpack_bf16x2(w[e]);
                    sum += f.x + f.y;
                    sq = fmaf(f.x, f.x, fmaf(f.y, f.y, sq));
                }
            }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        sum += __shfl_xor_sync(0xffffffffu, sum, o);
        sq += __shfl_xor_sync(0xffffffffu, sq, o);
    }
    __syncthreads();                                // modulation vectors staged
    if (!active) return;
    const float mean = sum / (float)H;
    const float var = fmaxf(sq / (float)H - mean * mean, 0.f);
    const float rstd = rsqrtf(var + 1e-6f);
    const bool staged = (b == b0);
    const uint4* sh_g = reinterpret_cast<const uint4*>(P.shift + (long long)b * mod_stride);
    const uint4* sc_g = reinterpret_cast<const uint4*>(P.scale + (long long)b * mod_stride);
    // modulate in place (v <- bf16(y), the value the bf16 path would hand to the GEMM), tracking the row's max |y|
    float amax = 0.f;
#pragma unroll
    for (int c = 0; c < kChunks; ++c)
        if (c < nchunks) {
            const int vi = c * 32 + lane;
            const uint4 hu = staged ? ln_smem[vi] : __ldg(sh_g + vi);
            const uint4 su = staged ? ln_smem[nvec + vi] : __ldg(sc_g + vi);
            const uint32_t xw[4] = {v[c].x, v[c].y, v[c].z, v[c].w};
            const uint32_t sw[4] = {su.x, su.y, su.z, su.w};
            const uint32_t hw[4] = {hu.x, hu.y, hu.z, hu.w};
            uint32_t ow[4];
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                float2 xf = unpack_bf16x2(xw[e]);
                float2 s2 = unpack_bf16x2(sw[e]);
                float2 h2 = unpack_bf16x2(hw[e]);
                float a0 = bf16_round(1.0f + s2.x), a1 = bf16_round(1.0f + s2.y);
                float n0 = (xf.x - mean) * rstd, n1 = (xf.y - mean) * rstd;
                const float y0 = __fadd_rn(__fmul_rn(a0, n0), h2.x), y1 = __fadd_rn(__fmul_rn(a1, n1), h2.y);
                ow[e] = pack_bf16x2(y0, y1);
                const float2 yr2 = unpack_bf16x2(ow[e]);                 // the scale refers to the bf16 values that get quantised
                amax = fmaxf(amax, fmaxf(fabsf(yr2.x), fabsf(yr2.y)));
            }
            v[c] = make_uint4(ow[0], ow[1], ow[2], ow[3]);
        }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
    const float s = fmaxf(amax, 1e-12f) * (1.0f / 448.0f);
    const float inv = 1.0f / s;
    if (lane == 0) P.row_scale[prow] = s;
    uint8_t* yr = P.y8 + prow * ldy;
#pragma unroll
    for (int c = 0; c < kChunks; ++c)
        if (c < nchunks) {
            const float2 f0 = unpack_bf16x2(v[c].x), f1 = unpack_bf16x2(v[c].y), f2 = unpack_bf16x2(v[c].z), f3 = unpack_bf16x2(v[c].w);
            uint2 o;
            o.x = pack_e4m3x4(f0.x * inv, f0.y * inv, f1.x * inv, f1.y * inv);
            o.y = pack_e4m3x4(f2.x * inv, f2.y * inv, f3.x * inv, f3.y * inv);
            *reinterpret_cast<uint2*>(yr + c * 256 + lane * 8) = o;
        }
}

// Row-wise e4m3 quantisation of a bf16 matrix that a GEMM epilogue or the attention kernel produced (fp8 level 2: the A operands
// of proj / mlp.2 / linear2).  One block per row: the row (<= 15360 elements) stays in registers between the max|x| reduction and
// the conversion, so the matrix is read once and the e4m3 copy written once.  Same scale rule as the fp8 LayerNorm:
// s = max(max|x|, 1e-12) / 448,  y8 = e4m3_rn_satfinite(x * (1 / s)).
constexpr int kQuantThreads = 192;
constexpr int kQuantMaxChunks = 10;                  // 16-byte chunks per thread: K <= 192 * 10 * 8 = 15360
__global__ void __launch_bounds__(kQuantThreads, 4)
quantize_rows_e4m3_kernel(const __nv_bfloat16* __restrict__ x, long long ldx, uint8_t* __restrict__ y8, long long ld8,
                          float* __restrict__ row_scale, int K) {
    __shared__ float red[kQuantThreads / 32];
    pdl_launch_dependents();
    pdl_wait();
    const long long row = blockIdx.x;
    const int nvec = K >> 3;
    const uint4* xr = reinterpret_cast<const uint4*>(x + row * ldx);
    uint4 v[kQuantMaxChunks];
    float amax = 0.f;
#pragma unroll
    for (int c = 0; c < kQuantMaxChunks; ++c) {
        const int idx = c * kQuantThreads + (int)threadIdx.x;
        if (idx < nvec) v[c] = xr[idx];
    }
#pragma unroll
    for (int c = 0; c < kQuantMaxChunks; ++c) {
        const int idx = c * kQuantThreads + (int)threadIdx.x;
        if (idx < nvec) {
            const uint32_t w[4] = {v[c].x, v[c].y, v[c].z, v[c].w};
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const float2 f = unpack_bf16x2(w[e]);
                amax = fmaxf(amax, fmaxf(fabsf(f.x), fabsf(f.y)));
            }
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = amax;
    __syncthreads();
#pragma unroll
    for (int w = 0; w < kQuantThreads / 32; ++w) amax = fmaxf(amax, red[w]);
    const float s = fmaxf(amax, 1e-12f) * (1.0f / 448.0f);
    const float inv = 1.0f / s;
    if (threadIdx.x == 0) row_scale[row] = s;
    uint8_t* yr = y8 + row * ld8;
#pragma unroll
    for (int c = 0; c < kQuantMaxChunks; ++c) {
        const int idx = c * kQuantThreads + (int)threadIdx.x;
        if (idx < nvec) {
            const float2 f0 = unpack_bf16x2(v[c].x), f1 = unpack_bf16x2(v[c].y), f2 = unpack_bf16x2(v[c].z), f3 = unpack_bf16x2(v[c].w);
            uint2 o;
            o.x = pack_e4m3x4(f0.x * inv, f0.y * inv, f1.x * inv, f1.y * inv);
            o.y = pack_e4m3x4(f2.x * inv, f2.y * inv, f3.x * inv, f3.y * inv);
            *reinterpret_cast<uint2*>(yr + (long long)idx * 8) = o;
        }
    }
}

// FP8 + statistics from the producer: with (sum, sum of squares) supplied by the GATE_RES epilogue the fp8 LayerNorm needs no
// register-resident row either -- pass A streams the row for max|bf16(y)|, pass B re-reads it (L1 / L2) and writes the e4m3 bytes.
// 48 registers -> 5 blocks per SM: one round at cfg B (the register-resident kernel above: 3 blocks per SM, two rounds).
__global__ void __launch_bounds__(kLnWarps * 32, 5)
ln_modulate_fp8_stats_kernel(const LnFp8Problem p0, const LnFp8Problem p1, const float2* stats0, const float2* stats1, int n_slots,
                             long long ldx, long long ldy, long long mod_stride, int H, int batch_rows) {
    extern __shared__ float4 ln_smem4[];
    pdl_launch_dependents();
    pdl_wait();
    const bool second = (int)blockIdx.x >= p0.blocks;
    const LnFp8Problem& P = second ? p1 : p0;
    const float2* stats = second ? stats1 : stats0;
    const int rows = P.rows, rows_per_batch = P.rows_per_batch;
    const int row0 = ((int)blockIdx.x - (second ? p0.blocks : 0)) * kLnWarps;
    const int b0 = row0 / rows_per_batch;
    const int nvec = H >> 3;
    const int row = row0 + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    const int nchunks = H >> 8;
    const bool active = row < rows;
    const int b = active ? row / rows_per_batch : b0;
    const long long prow = (long long)b * batch_rows + (row - b * rows_per_batch);
    float sum = 0.f, sq = 0.f;
    if (active) {
        const float2* st = stats + prow * n_slots;
        for (int i = lane; i < n_slots; i += 32) {
            const float2 v = __ldg(st + i);
            sum += v.x;
            sq += v.y;
        }
    }
    for (int i = threadIdx.x; i < nvec; i += blockDim.x) {
        const uint4 su = __ldg(reinterpret_cast<const uint4*>(P.scale + (long long)b0 * mod_stride) + i);
        const uint4 hu = __ldg(reinterpret_cast<const uint4*>(P.shift + (long long)b0 * mod_stride) + i);
        const float2 s0 = unpack_bf16x2(su.x), s1 = unpack_bf16x2(su.y), s2 = unpack_bf16x2(su.z), s3 = unpack_bf16x2(su.w);
        const float2 h0 = unpack_bf16x2(hu.x), h1 = unpack_bf16x2(hu.y), h2 = unpack_bf16x2(hu.z), h3 = unpack_bf16x2(hu.w);
        ln_smem4[i] = make_float4(bf16_round(1.0f + s0.x), bf16_round(1.0f + s0.y), bf16_round(1.0f + s1.x), bf16_round(1.0f + s1.y));
        ln_smem4[nvec + i] = make_float4(bf16_round(1.0f + s2.x), bf16_round(1.0f + s2.y), bf16_round(1.0f + s3.x), bf16_round(1.0f + s3.y));
        ln_smem4[2 * nvec + i] = make_float4(h0.x, h0.y, h1.x, h1.y);
        ln_smem4[3 * nvec + i] = make_float4(h2.x, h2.y, h3.x, h3.y);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        sum += __shfl_xor_sync(0xffffffffu, sum, o);
        sq += __shfl_xor_sync(0xffffffffu, sq, o);
    }
    __syncthreads();
    if (!active) return;
    const float mean = sum / (float)H;
    const float var = fmaxf(sq / (float)H - mean * mean, 0.f);
    const float rstd = rsqrtf(var + 1e-6f);
    const bool staged = (b == b0);
    const uint4* sh_g = reinterpret_cast<const uint4*>(P.shift + (long long)b * mod_stride);
    const uint4* sc_g = reinterpret_cast<const uint4*>(P.scale + (long long)b * mod_stride);
    const uint4* xr = reinterpret_cast<const uint4*>(P.x + prow * ldx) + lane;
    // the modulated values of one 8-element group, rounded to bf16 like the bf16 path rounds them
    auto group = [&](int c, float (&y)[8]) {
        const int vi = c * 32 + lane;
        const uint4 xv = xr[c * 32];
        float4 a0, a1, h0, h1;
        if (staged) {
            a0 = ln_smem4[vi]; a1 = ln_smem4[nvec + vi]; h0 = ln_smem4[2 * nvec + vi]; h1 = ln_smem4[3 * nvec + vi];
        } else {
            const uint4 su = __ldg(sc_g + vi), hu = __ldg(sh_g + vi);
            const float2 s0 = unpack_bf16x2(su.x), s1 = unpack_bf16x2(su.y), s2 = unpack_bf16x2(su.z), s3 = unpack_bf16x2(su.w);
            const float2 g0 = unpack_bf16x2(hu.x), g1 = unpack_bf16x2(hu.y), g2 = unpack_bf16x2(hu.z), g3 = unpack_bf16x2(hu.w);
            a0 = make_float4(bf16_round(1.0f + s0.x), bf16_round(1.0f + s0.y), bf16_round(1.0f + s1.x), bf16_round(1.0f + s1.y));
            a1 = make_float4(bf16_round(1.0f + s2.x), bf16_round(1.0f + s2.y), bf16_round(1.0f + s3.x), bf16_round(1.0f + s3.y));
            h0 = make_float4(g0.x, g0.y, g1.x, g1.y);
            h1 = make_float4(g2.x, g2.y, g3.x, g3.y);
        }
        const float av[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
        const float hv[8] = {h0.x, h0.y, h0.z, h0.w, h1.x, h1.y, h1.z, h1.w};
        const uint32_t xw[4] = {xv.x, xv.y, xv.z, xv.w};
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const float2 xf = unpack_bf16x2(xw[e]);
            const float n0 = (xf.x - mean) * rstd, n1 = (xf.y - mean) * rstd;
            y[2 * e] = bf16_round(__fadd_rn(__fmul_rn(av[2 * e], n0), hv[2 * e]));
            y[2 * e + 1] = bf16_round(__fadd_rn(__fmul_rn(av[2 * e + 1], n1), hv[2 * e + 1]));
        }
    };
    float amax = 0.f;
#pragma unroll 2
    for (int c = 0; c < nchunks; ++c) {
        float y[8];
        group(c, y);
#pragma unroll
        for (int e = 0; e < 8; ++e) amax = fmaxf(amax, fabsf(y[e]));
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
    const float s = fmaxf(amax, 1e-12f) * (1.0f / 448.0f);
    const float inv = 1.0f / s;
    if (lane == 0) P.row_scale[prow] = s;
    uint8_t* yr = P.y8 + prow * ldy;
#pragma unroll 2
    for (int c = 0; c < nchunks; ++c) {
        float y[8];
        group(c, y);
        uint2 o;
        o.x = pack_e4m3x4(y[0] * inv, y[1] * inv, y[2] * inv, y[3] * inv);
        o.y = pack_e4m3x4(y[4] * inv, y[5] * inv, y[6] * inv, y[7] * inv);
        *reinterpret_cast<uint2*>(yr + c * 256 + lane * 8) = o;
    }
}

// ------------------------------------------------------------------------------------------------
// small per-step / per-image helpers
// ------------------------------------------------------------------------------------------------
// Sinusoidal embedding (layers.py:28-49): out[n, 0:128] = cos(t * f), out[n, 128:256] = sin(t * f), bf16.
// `t_scaled` already holds time_factor * t in the dtype the reference computes it in (fp32 for timesteps,
// bf16-rounded for guidance); freqs[128] is computed on the host exactly like the reference does.
__global__ void timestep_embedding_kernel(const float* __restrict__ t_scaled, const float* __restrict__ freqs,
                                          __nv_bfloat16* __restrict__ out, int n) {
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= n * 128) return;
    const int r = idx >> 7, i = idx & 127;
    const float a = __fmul_rn(t_scaled[r], freqs[i]);
    out[r * 256 + i] = __float2bfloat16_rn(cosf(a));
    out[r * 256 + 128 + i] = __float2bfloat16_rn(sinf(a));
}

// y = silu(x) elementwise, bf16 -> bf16 (fp32 math), n % 2 == 0
__global__ void silu_kernel(const __nv_bfloat16* __restrict__ x, __nv_bfloat16* __restrict__ y, long long n) {
    const long long i = ((long long)blockIdx.x * blockDim.x + threadIdx.x) * 2;
    if (i >= n) return;
    float2 f = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(x + i));
    f.x = f.x / (1.0f + expf(-f.x));
    f.y = f.y / (1.0f + expf(-f.y));
    *reinterpret_cast<uint32_t*>(y + i) = pack_bf16x2(f.x, f.y);
}

// vec[r, :] = bf16(bf16(a[ra, :] + b[rb, :]) + c[rc, :]) with row maps r -> (r / a_div, r % b_mod ...) kept simple:
// a is indexed by r, b by r % b_rows, c by r % c_rows  (model.py:102-107: time + guidance + vector embeddings)
__global__ void add3_kernel(const __nv_bfloat16* __restrict__ a, const __nv_bfloat16* __restrict__ b, int b_rows,
                            const __nv_bfloat16* __restrict__ c, int c_rows, __nv_bfloat16* __restrict__ out, int rows,
                            int H) {
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (long long)rows * H) return;
    const int r = idx / H, col = idx % H;
    float s = __bfloat162float(a[idx]);
    if (b) s = bf16_round(s + __bfloat162float(b[(long long)(r % b_rows) * H + col]));
    if (c) s = bf16_round(s + __bfloat162float(c[(long long)(r % c_rows) * H + col]));
    out[idx] = __float2bfloat16_rn(s);
}

// RoPE table (layers.py:11-25, math.py:102-109): ids [rows, 3] fp32 -> (cos, sin), fp64 math like the reference.
// axes (16, 56, 56) -> 8 + 28 + 28 frequency pairs.  Output is PAIR-MAJOR [64][rows]: the GEMM epilogue's threads own
// consecutive rows, so a warp reads 32 consecutive float2 per pair (coalesced) instead of 32 strided cache lines.
__global__ void rope_table_kernel(const float* __restrict__ ids, float2* __restrict__ out, int rows, int d0, int d1,
                                  int d2, double theta) {
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    const int half = (d0 + d1 + d2) / 2;
    if (idx >= rows * half) return;
    const int r = idx / half;
    int i = idx % half;
    int axis, dim;
    if (i < d0 / 2) { axis = 0; dim = d0; }
    else if (i < (d0 + d1) / 2) { axis = 1; dim = d1; i -= d0 / 2; }
    else { axis = 2; dim = d2; i -= (d0 + d1) / 2; }
    const double scale = (double)(2 * i) / (double)dim;
    const double omega = 1.0 / pow(theta, scale);
    const double ang = (double)ids[r * 3 + axis] * omega;
    out[(long long)(idx % half) * rows + r] = make_float2((float)cos(ang), (float)sin(ang));
}

// Euler update (torchdiffeq fixed-grid euler via transport/integrators.py:119; SURVEY.md 8a-12):
//   x_new = bf16(x + bf16(dt_bf16 * (-v)))   (the sampler negates the model output, transport.py:384)
// Writes x_new to the trajectory slot and to columns [0, C) of the next model input (whose columns [C, ld_in) hold
// the constant `cond`, transport.py:194-196).
__global__ void euler_update_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ v,
                                    float dt_bf16, __nv_bfloat16* __restrict__ x_new, __nv_bfloat16* __restrict__ model_in,
                                    long long ld_in, long long rows, int C) {
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= rows * C) return;
    const long long r = idx / C;
    const int c = idx % C;
    const float f = -__bfloat162float(v[idx]);
    const float upd = bf16_round(dt_bf16 * f);
    const __nv_bfloat16 o = __float2bfloat16_rn(__bfloat162float(x[idx]) + upd);
    x_new[idx] = o;
    if (model_in) model_in[r * ld_in + c] = o;
}

// copy a [rows, C] bf16 matrix into columns [col0, col0 + C) of a wider matrix
__global__ void copy_cols_kernel(const __nv_bfloat16* __restrict__ src, long long lds, __nv_bfloat16* __restrict__ dst,
                                 long long ldd, int col0, long long rows, int C) {
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= rows * C) return;
    const long long r = idx / C;
    const int c = idx % C;
    dst[r * ldd + col0 + c] = src[r * lds + c];
}

}  // namespace vcb
