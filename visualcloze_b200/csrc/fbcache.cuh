// fbcache.cuh -- kernels of the opt-in first-block cache of the FLUX-DiT engine (vcb_flux_set_first_block_cache).
//
// After double block 0 the engine compares the img-row residual of that block, r_k = bf16(x1 - x0), with the one of the last
// computed evaluation, r_ref: diff = sum|r_k - r_ref| / sum|r_ref| over the valid img rows of every sample of a decision group
// (per-batch mode: one group, the whole batch; per-sample mode: one group per sample).  A skipped evaluation then writes
// x = bf16(x1 + R), R = x_final - x1 (fp32) of the last computed evaluation, and goes straight to the final layer.  Buffers are
// [B * Li, H] (row r = b * Li + i); x itself is the joint [B, L, H] residual stream.
#pragma once
#include <cuda_bf16.h>

#include <cstdint>

#include "host_util.cuh"

namespace vcb {

constexpr int kFbcWarps = 8;            // one warp per img row, 8 rows per CTA
constexpr int kFbcMaxBlocks = 1024;     // CTAs of the partial-sum pass = number of partial-sum slots
constexpr int kFbcThreads = 256;        // elementwise residual kernels
constexpr int kFbcDecideWarps = 8;      // decision kernel: one warp per group, groups strided over the warps

struct FbcRows {
    int B, Li, Lt, L, H;
    const int32_t* seqlens;             // [B] valid tokens of the joint sequence (Lt + valid img rows) or NULL
};

// the img rows of sample b that count for the decision: right-padded rows are excluded
__device__ __forceinline__ int fbc_valid_rows(const FbcRows& g, int b) {
    if (!g.seqlens) return g.Li;
    return min(max(g.seqlens[b] - g.Lt, 0), g.Li);
}

__device__ __forceinline__ int64_t fbc_x_row(const FbcRows& g, int r) {
    const int b = r / g.Li;
    return (int64_t)b * g.L + g.Lt + (r - b * g.Li);
}

// Pass 1.  Every row: r_k = bf16(x1 - x0) overwrites the x0 copy.  Valid rows (not when `first`: there is no r_ref yet): each CTA
// sums num = sum|r_k - r_ref| and den = sum|r_ref| in fp32 into its slot part[blockIdx.x].  The grid is `groups` equal runs of
// CTAs, run k covering the rows of group k only (groups = 1: every row; groups = B: sample k), so no slot straddles two groups.
// Fixed order -- a lane walks its columns row by row, the lanes of a warp combine by a butterfly, the warps in index order -- so
// equal inputs give equal sums, and one group of nb CTAs sums exactly as the per-batch pass of nb CTAs does.
__global__ void __launch_bounds__(kFbcWarps * 32) fbc_partial_kernel(__nv_bfloat16* __restrict__ x0_rk, const __nv_bfloat16* __restrict__ x,
                                                                     const __nv_bfloat16* __restrict__ r_ref, FbcRows g, int first,
                                                                     int groups, float2* __restrict__ part) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int nbs = gridDim.x / groups, grp = blockIdx.x / nbs, blk = blockIdx.x - grp * nbs;
    const int rows = g.B * g.Li / groups, r0 = grp * rows, nv = g.H / 8;
    float num = 0.f, den = 0.f;
    for (int k = blk * kFbcWarps + warp; k < rows; k += nbs * kFbcWarps) {
        const int r = r0 + k;
        const bool count = !first && (r % g.Li) < fbc_valid_rows(g, r / g.Li);
        uint4* a = reinterpret_cast<uint4*>(x0_rk + (int64_t)r * g.H);
        const uint4* c = reinterpret_cast<const uint4*>(x + fbc_x_row(g, r) * g.H);
        const uint4* q = reinterpret_cast<const uint4*>(r_ref + (int64_t)r * g.H);
        for (int v = lane; v < nv; v += 32) {
            uint4 va = a[v];
            const uint4 vc = c[v];
            __nv_bfloat162* pa = reinterpret_cast<__nv_bfloat162*>(&va);
            const __nv_bfloat162* pc = reinterpret_cast<const __nv_bfloat162*>(&vc);
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const float2 f0 = __bfloat1622float2(pa[j]), f1 = __bfloat1622float2(pc[j]);
                pa[j] = __floats2bfloat162_rn(f1.x - f0.x, f1.y - f0.y);
            }
            a[v] = va;
            if (count) {
                const uint4 vq = q[v];
                const __nv_bfloat162* pq = reinterpret_cast<const __nv_bfloat162*>(&vq);
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const float2 k = __bfloat1622float2(pa[j]), f = __bfloat1622float2(pq[j]);
                    num += fabsf(k.x - f.x) + fabsf(k.y - f.y);
                    den += fabsf(f.x) + fabsf(f.y);
                }
            }
        }
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) {
        num += __shfl_xor_sync(0xffffffffu, num, o);
        den += __shfl_xor_sync(0xffffffffu, den, o);
    }
    __shared__ float2 s[kFbcWarps];
    if (lane == 0) s[warp] = make_float2(num, den);
    __syncthreads();
    if (threadIdx.x == 0) {
        float2 t = s[0];
        for (int w = 1; w < kFbcWarps; ++w) { t.x += s[w].x; t.y += s[w].y; }
        part[blockIdx.x] = t;
    }
}

// Pass 2: warp w decides groups w, w + warps, ...; group k sums its nbs slots in a fixed order -> out[4k..4k+3] = {num, den, diff,
// skip}; diff = num / den (+inf when `first`), skip = !first && diff < threshold (a NaN diff -- no residual to compare with --
// computes).  out[4 * groups] = the number of groups that skip (groups = all skipped, 0 = none).
__global__ void __launch_bounds__(kFbcDecideWarps * 32) fbc_decide_kernel(const float2* __restrict__ part, int nbs, int groups,
                                                                          float threshold, int first, float* __restrict__ out) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int grp = warp; grp < groups; grp += blockDim.x >> 5) {
        const float2* p = part + grp * nbs;
        float num = 0.f, den = 0.f;
        for (int k = lane; k < nbs; k += 32) { num += p[k].x; den += p[k].y; }
#pragma unroll
        for (int o = 16; o; o >>= 1) {
            num += __shfl_xor_sync(0xffffffffu, num, o);
            den += __shfl_xor_sync(0xffffffffu, den, o);
        }
        if (lane == 0) {
            const float diff = first ? INFINITY : num / den;
            float* o = out + 4 * grp;
            o[0] = num; o[1] = den; o[2] = diff;
            o[3] = (!first && diff < threshold) ? 1.f : 0.f;
        }
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        int n = 0;
        for (int k = 0; k < groups; ++k) n += out[4 * k + 3] != 0.f;
        out[4 * groups] = (float)n;
    }
}

// computed evaluation, after the last block: R = x_final - x1 in fp32 (x1c = the saved img rows after block 0)
__global__ void __launch_bounds__(kFbcThreads) fbc_store_residual_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ x1c,
                                                                         float* __restrict__ R, FbcRows g) {
    const int nv = g.H / 8;
    const int64_t n = (int64_t)g.B * g.Li * nv;
    for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < n; t += (int64_t)gridDim.x * blockDim.x) {
        const int r = (int)(t / nv), v = (int)(t - (int64_t)r * nv);
        const uint4 vx = reinterpret_cast<const uint4*>(x + fbc_x_row(g, r) * g.H)[v];
        const uint4 v1 = reinterpret_cast<const uint4*>(x1c + (int64_t)r * g.H)[v];
        const __nv_bfloat162* px = reinterpret_cast<const __nv_bfloat162*>(&vx);
        const __nv_bfloat162* p1 = reinterpret_cast<const __nv_bfloat162*>(&v1);
        float4* o = reinterpret_cast<float4*>(R + (int64_t)r * g.H + 8 * v);
        float d[8];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const float2 a = __bfloat1622float2(px[j]), b = __bfloat1622float2(p1[j]);
            d[2 * j] = a.x - b.x;
            d[2 * j + 1] = a.y - b.y;
        }
        o[0] = make_float4(d[0], d[1], d[2], d[3]);
        o[1] = make_float4(d[4], d[5], d[6], d[7]);
    }
}

// skipped evaluation: the img rows of x (= x1) become bf16(x1 + R)
__global__ void __launch_bounds__(kFbcThreads) fbc_apply_residual_kernel(__nv_bfloat16* __restrict__ x, const float* __restrict__ R, FbcRows g) {
    const int nv = g.H / 8;
    const int64_t n = (int64_t)g.B * g.Li * nv;
    for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < n; t += (int64_t)gridDim.x * blockDim.x) {
        const int r = (int)(t / nv), v = (int)(t - (int64_t)r * nv);
        uint4* px = reinterpret_cast<uint4*>(x + fbc_x_row(g, r) * g.H) + v;
        uint4 vx = *px;
        __nv_bfloat162* p = reinterpret_cast<__nv_bfloat162*>(&vx);
        const float4* q = reinterpret_cast<const float4*>(R + (int64_t)r * g.H + 8 * v);
        const float4 r0 = q[0], r1 = q[1];
        const float add[8] = {r0.x, r0.y, r0.z, r0.w, r1.x, r1.y, r1.z, r1.w};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const float2 a = __bfloat1622float2(p[j]);
            p[j] = __floats2bfloat162_rn(a.x + add[2 * j], a.y + add[2 * j + 1]);
        }
        *px = vx;
    }
}

// CTAs of one group's partial-sum run: enough for one warp per row, at most kFbcMaxBlocks over all groups
inline int fbc_group_blocks(const FbcRows& g, int groups) {
    const int need = (g.B * g.Li / groups + kFbcWarps - 1) / kFbcWarps, cap = kFbcMaxBlocks / groups;
    return need < cap ? need : cap;
}

// both passes of the decision for `groups` (1 or B) groups; `res` [4 * groups + 1] fp32 device, `part` [kFbcMaxBlocks] float2 device
inline int fbc_decide(uint16_t* x0_rk, const uint16_t* x, const uint16_t* r_ref, const FbcRows& g, int groups, bool first, float threshold,
                      float2* part, float* res, cudaStream_t st) {
    const int nbs = fbc_group_blocks(g, groups);
    {
        ProfScope prof(PROF_OTHER, st);
        fbc_partial_kernel<<<nbs * groups, kFbcWarps * 32, 0, st>>>(reinterpret_cast<__nv_bfloat16*>(x0_rk), reinterpret_cast<const __nv_bfloat16*>(x),
                                                                    reinterpret_cast<const __nv_bfloat16*>(r_ref), g, first ? 1 : 0, groups, part);
        if (int rc = check_launch("fbc_partial")) return rc;
    }
    ProfScope prof(PROF_OTHER, st);
    const int warps = groups < kFbcDecideWarps ? groups : kFbcDecideWarps;
    fbc_decide_kernel<<<1, warps * 32, 0, st>>>(part, nbs, groups, threshold, first ? 1 : 0, res);
    return check_launch("fbc_decide");
}

inline unsigned fbc_elementwise_blocks(const FbcRows& g) {
    const int64_t n = (int64_t)g.B * g.Li * (g.H / 8);
    const int64_t b = (n + kFbcThreads - 1) / kFbcThreads;
    return (unsigned)(b < 4096 ? b : 4096);
}

inline int fbc_store_residual(const uint16_t* x, const uint16_t* x1c, float* R, const FbcRows& g, cudaStream_t st) {
    ProfScope prof(PROF_OTHER, st);
    fbc_store_residual_kernel<<<fbc_elementwise_blocks(g), kFbcThreads, 0, st>>>(reinterpret_cast<const __nv_bfloat16*>(x),
                                                                                 reinterpret_cast<const __nv_bfloat16*>(x1c), R, g);
    return check_launch("fbc_store_residual");
}

inline int fbc_apply_residual(uint16_t* x, const float* R, const FbcRows& g, cudaStream_t st) {
    ProfScope prof(PROF_OTHER, st);
    fbc_apply_residual_kernel<<<fbc_elementwise_blocks(g), kFbcThreads, 0, st>>>(reinterpret_cast<__nv_bfloat16*>(x), R, g);
    return check_launch("fbc_apply_residual");
}

}  // namespace vcb
