// elementwise.cuh -- HBM-bound helpers of the FLUX-DiT step (coalesced 16-byte accesses, fp32 math).
#pragma once
#include <type_traits>

#include "vcb_common.cuh"

namespace vcb {

// ------------------------------------------------------------------------------------------------
// AdaLN: y = bf16( bf16(1 + scale) * LayerNorm(x) + shift ), LayerNorm without affine, eps 1e-6, fp32 stats.
// Replaces F.layer_norm + two elementwise passes + the autocast cast (layers.py:163-164,191,195,234,257).
// Algorithmic bytes: read + write of [rows, H] bf16 = 4*rows*H bytes.
//
// One warp per row, 8 rows per block.  One launch may carry two problems (the img and txt streams of a DoubleStreamBlock,
// layers.py:163 / 170): blocks [0, p0.blocks) work on p0, the rest on p1.  One body, ln_modulate_body<kStats, kFp8>, serves
// four entry points:
//   statistics  kStats = false: a pass over the row (sum and sum of squares in fp32);
//               kStats = true:  the GATE_RES epilogue of the GEMM that wrote x left one (sum, sum of squares) pair per 64
//                               columns (gemm_sm90.cuh, row_stats); a warp adds the row's n_slots pairs in a fixed order;
//   output      kFp8 = false: bf16 rows, one read-modulate-write pass;
//               kFp8 = true:  e4m3 bytes with ONE fp32 scale per row, s = max|bf16(y)| / 448, y8 = e4m3(bf16(y) / s) -- one
//                             pass for the max, then one that re-reads the row and writes the bytes.  The fp8 GEMM multiplies
//                             its accumulator by s (a_scale) again.
// No pass keeps the row in registers: the re-reads hit L1 / L2 (the warp has just touched those lines), and a small register
// footprint is what lets 4-5 blocks x 8 warps share an SM, so that every row of a cfg-B sequence (3968) is in flight in ONE round.
// ------------------------------------------------------------------------------------------------
constexpr int kLnWarps = 8;           // rows per block
constexpr int kLnMaxHidden = 6144;    // the staged modulation vectors take 8 * H bytes of the default 48 KB of dynamic shared memory

VCB_DEVICE uint32_t pack_e4m3x4(float a, float b, float c, float d) {
    uint16_t lo, hi;
    asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(lo) : "f"(b), "f"(a));      // first source -> upper byte
    asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(hi) : "f"(d), "f"(c));
    return (uint32_t)lo | ((uint32_t)hi << 16);
}

// Logical row (b, i) of a problem lives at physical row b * batch_rows + i of x and y (a stream inside a joint [B, L, H] buffer);
// stats and row_scale are indexed by the physical row too.
struct LnProblem {
    const __nv_bfloat16* x;
    void* y;                                        // bf16 rows, or e4m3 bytes
    float* row_scale;                               // e4m3 output: [physical rows]
    const float2* stats;                            // statistics from the producer: [physical rows][n_slots]
    const __nv_bfloat16* shift; const __nv_bfloat16* scale;
    int rows, rows_per_batch, blocks;
};

// 8 elements of the modulation row: a = bf16(1 + scale) (a bf16 op in the reference) and shift, as two float4 each
VCB_DEVICE void ln_mod8(uint4 su, uint4 hu, float4& a0, float4& a1, float4& h0, float4& h1) {
    const float2 s0 = unpack_bf16x2(su.x), s1 = unpack_bf16x2(su.y), s2 = unpack_bf16x2(su.z), s3 = unpack_bf16x2(su.w);
    const float2 g0 = unpack_bf16x2(hu.x), g1 = unpack_bf16x2(hu.y), g2 = unpack_bf16x2(hu.z), g3 = unpack_bf16x2(hu.w);
    a0 = make_float4(bf16_round(1.0f + s0.x), bf16_round(1.0f + s0.y), bf16_round(1.0f + s1.x), bf16_round(1.0f + s1.y));
    a1 = make_float4(bf16_round(1.0f + s2.x), bf16_round(1.0f + s2.y), bf16_round(1.0f + s3.x), bf16_round(1.0f + s3.y));
    h0 = make_float4(g0.x, g0.y, g1.x, g1.y);
    h1 = make_float4(g2.x, g2.y, g3.x, g3.y);
}

template <bool kStats, bool kFp8>
VCB_DEVICE void ln_modulate_body(const LnProblem& p0, const LnProblem& p1, long long ldx, long long ldy, long long mod_stride, int H,
                                 int batch_rows, int n_slots) {
    // loads in flight per lane in the output pass: the bf16 kernel with producer statistics runs at 4 blocks per SM and has the
    // registers for six, the others (5 blocks per SM) for two
    constexpr int kUnroll = kStats && !kFp8 ? 6 : 2;
    // [4][H / 8] float4: bf16(1 + scale) and shift of sample b0, converted ONCE per block -- group i (8 elements) of the
    // modulation row: a elements 0-3 at [i], 4-7 at [nvec + i]; shift at [2 nvec + i], [3 nvec + i] (consecutive lanes read
    // consecutive float4: no bank conflicts)
    extern __shared__ float4 ln_smem4[];
    pdl_launch_dependents();
    pdl_wait();
    const bool second = (int)blockIdx.x >= p0.blocks;
    const LnProblem P = second ? p1 : p0;              // by value: the fields are selected in registers, no stack copy
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
    float sum = 0.f, sq = 0.f;
    if (active) {
        if constexpr (kStats) {
            const float2* st = P.stats + prow * n_slots;
            for (int i = lane; i < n_slots; i += 32) {
                const float2 v = __ldg(st + i);
                sum += v.x;
                sq += v.y;
            }
        } else {                                    // four 16-byte loads in flight per lane (40 warps per SM keep ~80 KB in flight)
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
    }
    for (int i = threadIdx.x; i < nvec; i += blockDim.x)
        ln_mod8(__ldg(reinterpret_cast<const uint4*>(P.scale + (long long)b0 * mod_stride) + i),
                __ldg(reinterpret_cast<const uint4*>(P.shift + (long long)b0 * mod_stride) + i),
                ln_smem4[i], ln_smem4[nvec + i], ln_smem4[2 * nvec + i], ln_smem4[3 * nvec + i]);
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
    // the modulated fp32 values of 8-element group c of the row: the product and the sum are separate fp32 operations
    // (LayerNorm returns fp32, then (1 + scale) * ln + shift)
    auto group = [&](int c, float (&y)[8]) {
        const int vi = c * 32 + lane;
        const uint4 xv = xr[c * 32];
        float4 a0, a1, h0, h1;
        if (staged) {
            a0 = ln_smem4[vi]; a1 = ln_smem4[nvec + vi]; h0 = ln_smem4[2 * nvec + vi]; h1 = ln_smem4[3 * nvec + vi];
        } else {                                    // a block straddling two samples: this row's vectors straight from global
            ln_mod8(__ldg(sc_g + vi), __ldg(sh_g + vi), a0, a1, h0, h1);
        }
        const float av[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
        const float hv[8] = {h0.x, h0.y, h0.z, h0.w, h1.x, h1.y, h1.z, h1.w};
        const uint32_t xw[4] = {xv.x, xv.y, xv.z, xv.w};
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const float2 xf = unpack_bf16x2(xw[e]);
            const float n0 = (xf.x - mean) * rstd, n1 = (xf.y - mean) * rstd;
            y[2 * e] = __fadd_rn(__fmul_rn(av[2 * e], n0), hv[2 * e]);
            y[2 * e + 1] = __fadd_rn(__fmul_rn(av[2 * e + 1], n1), hv[2 * e + 1]);
        }
    };
    if constexpr (!kFp8) {
        uint4* yr = reinterpret_cast<uint4*>(static_cast<__nv_bfloat16*>(P.y) + prow * ldy) + lane;
#pragma unroll kUnroll
        for (int c = 0; c < nchunks; ++c) {
            float y[8];
            group(c, y);
            yr[c * 32] = make_uint4(pack_bf16x2(y[0], y[1]), pack_bf16x2(y[2], y[3]), pack_bf16x2(y[4], y[5]), pack_bf16x2(y[6], y[7]));
        }
    } else {
        // the scale refers to the bf16 values the bf16 path would hand to the GEMM: round before the max and the quantisation
        float amax = 0.f;
#pragma unroll kUnroll
        for (int c = 0; c < nchunks; ++c) {
            float y[8];
            group(c, y);
#pragma unroll
            for (int e = 0; e < 8; ++e) amax = fmaxf(amax, fabsf(bf16_round(y[e])));
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
        const float s = fmaxf(amax, 1e-12f) * (1.0f / 448.0f);
        const float inv = 1.0f / s;
        if (lane == 0) P.row_scale[prow] = s;
        uint8_t* yr = static_cast<uint8_t*>(P.y) + prow * ldy;
#pragma unroll kUnroll
        for (int c = 0; c < nchunks; ++c) {
            float y[8];
            group(c, y);
#pragma unroll
            for (int e = 0; e < 8; ++e) y[e] = bf16_round(y[e]) * inv;
            uint2 o;
            o.x = pack_e4m3x4(y[0], y[1], y[2], y[3]);
            o.y = pack_e4m3x4(y[4], y[5], y[6], y[7]);
            *reinterpret_cast<uint2*>(yr + c * 256 + lane * 8) = o;
        }
    }
}

// The four instantiations; each keeps the occupancy its variant was tuned for.  5 blocks x 8 warps per SM = 148 x 40 = 5920
// resident warps >= the 3968 rows of a cfg-B sequence.  The bf16 kernel with producer statistics trades a block for registers:
// 4 blocks per SM = 4736 warps are still one round, and 64 registers let a lane keep six 16-byte loads in flight -- that kernel
// is latency-bound (one dependent chain per warp), so the row is covered by two batches of loads instead of four.
__global__ void __launch_bounds__(kLnWarps * 32, 5)
ln_modulate2_kernel(const LnProblem p0, const LnProblem p1, long long ldx, long long ldy, long long mod_stride, int H, int batch_rows,
                    int n_slots) {
    ln_modulate_body<false, false>(p0, p1, ldx, ldy, mod_stride, H, batch_rows, n_slots);
}
__global__ void __launch_bounds__(kLnWarps * 32, 4)
ln_modulate_stats_kernel(const LnProblem p0, const LnProblem p1, long long ldx, long long ldy, long long mod_stride, int H, int batch_rows,
                         int n_slots) {
    ln_modulate_body<true, false>(p0, p1, ldx, ldy, mod_stride, H, batch_rows, n_slots);
}
__global__ void __launch_bounds__(kLnWarps * 32, 5)
ln_modulate_fp8_kernel(const LnProblem p0, const LnProblem p1, long long ldx, long long ldy, long long mod_stride, int H, int batch_rows,
                       int n_slots) {
    ln_modulate_body<false, true>(p0, p1, ldx, ldy, mod_stride, H, batch_rows, n_slots);
}
__global__ void __launch_bounds__(kLnWarps * 32, 5)
ln_modulate_fp8_stats_kernel(const LnProblem p0, const LnProblem p1, long long ldx, long long ldy, long long mod_stride, int H,
                             int batch_rows, int n_slots) {
    ln_modulate_body<true, true>(p0, p1, ldx, ldy, mod_stride, H, batch_rows, n_slots);
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

// ODE stage updates of torchdiffeq's fixed-grid solvers as transport/integrators.py:119 calls them (DESIGN.md 2e).  Every
// binary operation of the torch expression is one eager bf16 op: fp32 math on bf16 operands, one rounding r() per op.  The
// sampler negates the model output (transport.py:384), k_i = -v_i, which is exact.  `h` is the 0-dim fp32 time-step tensor as
// a bf16 tensor op sees it, bf16(dt) (SURVEY.md 8a-12) -- bf16(0.5 * dt) for the midpoint state; the Python-float constants
// 1/3, 3 and 0.125 enter the fp32 op math unrounded.
//   kOdeAxpy      r(y0 + r(h * k1))                                 euler; midpoint state (h = bf16(dt/2)) and final (k1 := k2)
//   kOdeRk4K2     r(y0 + r(r(h * k1) * 1/3))                        rk4: y0 + dt * k1 * _one_third
//   kOdeRk4K3     r(y0 + r(h * r(k2 - r(k1 * 1/3))))                rk4: y0 + dt * (k2 - k1 * _one_third)
//   kOdeRk4K4     r(y0 + r(h * r(r(k1 - k2) + k3)))                 rk4: y0 + dt * (k1 - k2 + k3)
//   kOdeRk4Final  r(y0 + r(r(h * r(r(k1 + r(3 r(k2 + k3))) + k4)) * 0.125))   rk4: y0 + (k1 + 3 * (k2 + k3) + k4) * dt * 0.125
// The result goes to y_out (a trajectory slot or a stage buffer) and, when model_in is set, to columns [0, C) of the next model
// input, whose columns [C, ld_in) hold the constant `cond` (transport.py:194-196).  kVec = 8: 16-byte accesses (C and ld_in
// multiples of 8, 16-byte aligned pointers); kVec = 1 takes any layout.
enum OdeForm : int { kOdeAxpy = 0, kOdeRk4K2, kOdeRk4K3, kOdeRk4K4, kOdeRk4Final };
constexpr int kOdeMaxV = 4;

struct OdeVs { const __nv_bfloat16* v[kOdeMaxV]; };

template <int kForm>
VCB_DEVICE float ode_stage_value(float y0, const float* k, float h) {
    constexpr float kThird = 1.0f / 3.0f;
    float d;
    if constexpr (kForm == kOdeAxpy) {
        d = bf16_round(h * k[0]);
    } else if constexpr (kForm == kOdeRk4K2) {
        d = bf16_round(bf16_round(h * k[0]) * kThird);
    } else if constexpr (kForm == kOdeRk4K3) {
        d = bf16_round(h * bf16_round(k[1] - bf16_round(k[0] * kThird)));
    } else if constexpr (kForm == kOdeRk4K4) {
        d = bf16_round(h * bf16_round(bf16_round(k[0] - k[1]) + k[2]));
    } else {
        const float s = bf16_round(3.0f * bf16_round(k[1] + k[2]));
        const float q = bf16_round(bf16_round(k[0] + s) + k[3]);
        d = bf16_round(bf16_round(q * h) * 0.125f);
    }
    return y0 + d;                                   // rounded by the caller's store
}

template <int kForm, int kVec>
__global__ void __launch_bounds__(256) ode_stage_kernel(const __nv_bfloat16* __restrict__ y0, OdeVs vs, float h,
                                                        __nv_bfloat16* __restrict__ y_out, __nv_bfloat16* __restrict__ model_in,
                                                        long long ld_in, long long rows, int C) {
    constexpr int kNv = kForm == kOdeAxpy ? 1 : kForm == kOdeRk4K2 ? 1 : kForm == kOdeRk4K3 ? 2 : kForm == kOdeRk4K4 ? 3 : 4;
    using Pack = std::conditional_t<kVec == 8, uint4, __nv_bfloat16>;
    const long long idx = ((long long)blockIdx.x * blockDim.x + threadIdx.x) * kVec;
    if (idx >= rows * C) return;
    const long long r = idx / C;
    const int c = (int)(idx % C);
    __nv_bfloat16 yv[kVec], vv[kNv][kVec], o[kVec];
    *reinterpret_cast<Pack*>(yv) = *reinterpret_cast<const Pack*>(y0 + idx);
#pragma unroll
    for (int i = 0; i < kNv; ++i) *reinterpret_cast<Pack*>(vv[i]) = *reinterpret_cast<const Pack*>(vs.v[i] + idx);
#pragma unroll
    for (int j = 0; j < kVec; ++j) {
        float k[kNv];
#pragma unroll
        for (int i = 0; i < kNv; ++i) k[i] = -__bfloat162float(vv[i][j]);
        o[j] = __float2bfloat16_rn(ode_stage_value<kForm>(__bfloat162float(yv[j]), k, h));
    }
    *reinterpret_cast<Pack*>(y_out + idx) = *reinterpret_cast<const Pack*>(o);
    if (model_in) *reinterpret_cast<Pack*>(model_in + r * ld_in + c) = *reinterpret_cast<const Pack*>(o);
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
