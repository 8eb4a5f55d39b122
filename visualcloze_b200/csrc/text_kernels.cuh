// text_kernels.cuh -- the non-GEMM pieces of the two text encoders behind models/modules/conditioner.py:5-37 (SURVEY.md 8f-4):
// T5 v1.1 encoder (HF T5EncoderModel: T5LayerNorm, relative-position-bias attention, gated GELU) and the CLIP-L text model
// (nn.LayerNorm, causal attention, quick-GELU).  Everything with a matrix in it goes through gemm_sm90.cuh; what is left is
// HBM-bound row work and a small attention (head_dim 64, at most 512 keys, 4.3 GFLOP per T5 layer) that runs on the CUDA cores.
// Rounding points follow the bf16 HF modules the reference loads (torch_dtype=torch.bfloat16, models/util.py:425-431).
#pragma once
#include "vcb_common.cuh"

namespace vcb {

// out[t, :] = table[ids[t], :] (+ pos_table[t % L, :], the CLIP position embedding; both adds in bf16 like nn.Embedding sums)
__global__ void embedding_kernel(const __nv_bfloat16* __restrict__ table, const long long* __restrict__ ids,
                                 const __nv_bfloat16* __restrict__ pos_table, __nv_bfloat16* __restrict__ out, long long ldo,
                                 long long n_tokens, int dim, int L, long long vocab) {
    const long long t = blockIdx.x;
    long long id = ids[t];
    id = id < 0 ? 0 : (id >= vocab ? vocab - 1 : id);
    const uint4* src = reinterpret_cast<const uint4*>(table + id * dim);
    const uint4* pos = pos_table ? reinterpret_cast<const uint4*>(pos_table + (t % L) * dim) : nullptr;
    uint4* dst = reinterpret_cast<uint4*>(out + t * ldo);
    for (int i = threadIdx.x; i < dim / 8; i += blockDim.x) {
        uint4 v = __ldg(src + i);
        if (pos) {
            const uint4 p = __ldg(pos + i);
            const uint32_t a[4] = {v.x, v.y, v.z, v.w}, b[4] = {p.x, p.y, p.z, p.w};
            uint32_t o[4];
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const float2 fa = unpack_bf16x2(a[e]), fb = unpack_bf16x2(b[e]);
                o[e] = pack_bf16x2(fa.x + fb.x, fa.y + fb.y);
            }
            v = make_uint4(o[0], o[1], o[2], o[3]);
        }
        dst[i] = v;
    }
}

// One warp per row.  kAffine = false: T5LayerNorm (modeling_t5.py): y = weight * bf16(x * rsqrt(mean(x^2) + eps)), no mean, no bias.
// kAffine = true: nn.LayerNorm on a bf16 tensor: fp32 statistics, y = bf16((x - mean) * rstd * weight + bias).
template <bool kAffine>
__global__ void __launch_bounds__(256)
rownorm_kernel(const __nv_bfloat16* __restrict__ x, long long ldx, const __nv_bfloat16* __restrict__ weight,
               const __nv_bfloat16* __restrict__ bias, __nv_bfloat16* __restrict__ y, long long ldy, long long rows, int dim, float eps) {
    const long long row = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (row >= rows) return;
    const uint4* xr = reinterpret_cast<const uint4*>(x + row * ldx);
    const int nvec = dim >> 3;
    float sum = 0.f, sq = 0.f;
    for (int i = lane; i < nvec; i += 32) {
        const uint4 v = xr[i];
        const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const float2 f = unpack_bf16x2(w[e]);
            sum += f.x + f.y;
            sq = fmaf(f.x, f.x, fmaf(f.y, f.y, sq));
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        sum += __shfl_xor_sync(0xffffffffu, sum, o);
        sq += __shfl_xor_sync(0xffffffffu, sq, o);
    }
    const float mean = kAffine ? sum / (float)dim : 0.f;
    const float var = kAffine ? fmaxf(sq / (float)dim - mean * mean, 0.f) : sq / (float)dim;
    const float rstd = rsqrtf(var + eps);
    const uint4* wr = reinterpret_cast<const uint4*>(weight);
    const uint4* br = reinterpret_cast<const uint4*>(bias);
    uint4* yr = reinterpret_cast<uint4*>(y + row * ldy);
    for (int i = lane; i < nvec; i += 32) {                 // second read of the row: L1 / L2 hits
        const uint4 v = xr[i], g = __ldg(wr + i);
        const uint4 bb = kAffine ? __ldg(br + i) : make_uint4(0, 0, 0, 0);
        const uint32_t xv[4] = {v.x, v.y, v.z, v.w}, gv[4] = {g.x, g.y, g.z, g.w}, bv[4] = {bb.x, bb.y, bb.z, bb.w};
        uint32_t o[4];
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const float2 f = unpack_bf16x2(xv[e]), w2 = unpack_bf16x2(gv[e]), b2 = unpack_bf16x2(bv[e]);
            if constexpr (kAffine) {
                o[e] = pack_bf16x2(fmaf((f.x - mean) * rstd, w2.x, b2.x), fmaf((f.y - mean) * rstd, w2.y, b2.y));
            } else {
                // fp32 product, cast to bf16, then the bf16 multiply by the weight
                o[e] = pack_bf16x2(w2.x * bf16_round(f.x * rstd), w2.y * bf16_round(f.y * rstd));
            }
        }
        yr[i] = make_uint4(o[0], o[1], o[2], o[3]);
    }
}

// T5DenseGatedActDense: out = gelu_new(a) * b with a = ab[:, :dff], b = ab[:, dff:] (wi_0 and wi_1 share one GEMM).
// NewGELUActivation on a bf16 tensor: 0.5 x (1 + tanh(sqrt(2/pi) (x + 0.044715 x^3))); evaluated in fp32 and rounded once.
__global__ void gated_gelu_kernel(const __nv_bfloat16* __restrict__ ab, long long ld, __nv_bfloat16* __restrict__ out, long long ldo,
                                  long long rows, int dff) {
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const int nvec = dff >> 3;
    if (idx >= rows * nvec) return;
    const long long row = idx / nvec;
    const int c = (int)(idx - row * nvec);
    const uint4 a = *reinterpret_cast<const uint4*>(ab + row * ld + c * 8);
    const uint4 b = *reinterpret_cast<const uint4*>(ab + row * ld + dff + c * 8);
    const uint32_t av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {b.x, b.y, b.z, b.w};
    uint32_t o[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) {
        const float2 fa = unpack_bf16x2(av[e]), fb = unpack_bf16x2(bv[e]);
        o[e] = pack_bf16x2(bf16_round(gelu_tanh(fa.x)) * fb.x, bf16_round(gelu_tanh(fa.y)) * fb.y);
    }
    *reinterpret_cast<uint4*>(out + row * ldo + c * 8) = make_uint4(o[0], o[1], o[2], o[3]);
}

// CLIP's quick_gelu: x * sigmoid(1.702 x)
__global__ void quick_gelu_kernel(const __nv_bfloat16* __restrict__ x, __nv_bfloat16* __restrict__ y, long long n) {
    const long long i = ((long long)blockIdx.x * blockDim.x + threadIdx.x) * 2;
    if (i >= n) return;
    const float2 f = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(x + i));
    *reinterpret_cast<uint32_t*>(y + i) = pack_bf16x2(f.x / (1.0f + __expf(-1.702f * f.x)), f.y / (1.0f + __expf(-1.702f * f.y)));
}

// ------------------------------------------------------------------------------------------------
// Small attention: head_dim 64, L <= 512 keys, additive bias (T5: relative position bias, no 1/sqrt(d)) or scale + causal mask
// (CLIP).  One block (256 threads) = 32 query rows of one (sample, head); the head's K, then its V, live in ONE shared buffer.
//   stage K  16-byte global loads, eight in flight per thread before the first shared store (the loop is latency-bound otherwise)
//   phase 1  scores: thread t owns keys t%128 + {0, 128, 256, 384} and 16 of the rows: per dim pair one K load per key
//            (conflict-free: rows are padded to 66 elements) and 16 broadcast q loads feed 16 x 4 x 2 FMAs
//   stage V  over K (no longer needed), then
//   phase 2  softmax per row in fp32 (one warp per 4 rows), probabilities rounded to bf16 (HF: softmax(scores.float()).type_as)
//   phase 3  out: thread t owns row t / 8 and 8 head dims
// HF rounding points: scores = bf16(q k^T) [* scale], + bias in bf16, fp32 softmax, bf16 probabilities, fp32 PV sum, bf16 out.
// ------------------------------------------------------------------------------------------------
constexpr int kSaRows = 32;
constexpr int kSaThreads = 256;
constexpr int kSaMaxL = 512;
constexpr int kSaKStride = 66;     // bf16 elements per K row in shared memory (33 words: bank = key index)
struct SmallAttnParams {
    const __nv_bfloat16* q; const __nv_bfloat16* k; const __nv_bfloat16* v;   // row (b * L + i), head h at column h * 64
    long long ld;                   // row stride of q / k / v (elements)
    const __nv_bfloat16* bias;      // [heads, L, L] or null
    __nv_bfloat16* out; long long ldo;
    int L, heads; float scale; int causal;
};
inline size_t small_attn_smem(int L) {
    const int Lp = (L + 3) & ~3;
    return (size_t)Lp * kSaKStride * 2 + (size_t)kSaRows * Lp * 4 + (size_t)kSaRows * Lp * 2 + (size_t)kSaRows * 64 * 4;
}
__global__ void __launch_bounds__(kSaThreads)
small_attention_kernel(const SmallAttnParams p) {
    extern __shared__ uint8_t sa_smem[];
    const int L = p.L, Lp = (L + 3) & ~3;
    __nv_bfloat16* sKV = reinterpret_cast<__nv_bfloat16*>(sa_smem);                      // K [Lp][66], later V [Lp][64]
    float* sS = reinterpret_cast<float*>(sKV + (size_t)Lp * kSaKStride);                 // [32][Lp]
    __nv_bfloat16* sP = reinterpret_cast<__nv_bfloat16*>(sS + (size_t)kSaRows * Lp);     // [32][Lp]
    float* sQ = reinterpret_cast<float*>(sP + (size_t)kSaRows * Lp);                     // [32][64]
    const int row0 = blockIdx.x * kSaRows, h = blockIdx.y, b = blockIdx.z;
    const int tid = threadIdx.x;
    const long long base = (long long)b * L;
    const int pieces = Lp * 8;                                   // 16-byte pieces of one [Lp][64] operand
    // ---- stage K and the 32 query rows ----
    for (int i0 = tid; i0 < pieces; i0 += 8 * kSaThreads) {
        uint4 buf[8];
#pragma unroll
        for (int u = 0; u < 8; ++u) {
            const int i = i0 + u * kSaThreads, j = i >> 3, c = i & 7;
            buf[u] = (i < pieces && j < L) ? *reinterpret_cast<const uint4*>(p.k + (base + j) * p.ld + h * 64 + c * 8) : make_uint4(0, 0, 0, 0);
        }
#pragma unroll
        for (int u = 0; u < 8; ++u) {
            const int i = i0 + u * kSaThreads, j = i >> 3, c = i & 7;
            if (i < pieces) {
                uint32_t* kd = reinterpret_cast<uint32_t*>(sKV + (size_t)j * kSaKStride + c * 8);     // 4-byte aligned (66 * 2 = 132)
                kd[0] = buf[u].x; kd[1] = buf[u].y; kd[2] = buf[u].z; kd[3] = buf[u].w;
            }
        }
    }
    for (int i = tid; i < kSaRows * 64; i += kSaThreads) {
        const int r = i >> 6, d = i & 63;
        sQ[i] = (row0 + r < L) ? __bfloat162float(p.q[(base + row0 + r) * p.ld + h * 64 + d]) : 0.f;
    }
    __syncthreads();
    // ---- phase 1: scores ----
    {
        const int kt = tid & 127, rg = (tid >> 7) * 16;          // my keys kt + 128 u, my rows rg .. rg + 15
        float acc[16][4];
#pragma unroll
        for (int r = 0; r < 16; ++r)
#pragma unroll
            for (int u = 0; u < 4; ++u) acc[r][u] = 0.f;
#pragma unroll 4
        for (int d = 0; d < 64; d += 2) {
            float2 kf[4];
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                const int j = kt + u * 128;
                kf[u] = j < Lp ? unpack_bf16x2(*reinterpret_cast<const uint32_t*>(sKV + (size_t)j * kSaKStride + d)) : make_float2(0.f, 0.f);
            }
#pragma unroll
            for (int r = 0; r < 16; ++r) {
                const float2 qf = *reinterpret_cast<const float2*>(sQ + (rg + r) * 64 + d);
#pragma unroll
                for (int u = 0; u < 4; ++u) acc[r][u] = fmaf(qf.x, kf[u].x, fmaf(qf.y, kf[u].y, acc[r][u]));
            }
        }
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            const int j = kt + u * 128;
            if (j >= Lp) continue;
#pragma unroll
            for (int r = 0; r < 16; ++r) {
                const int i = row0 + rg + r;
                float s = bf16_round(acc[r][u]);                                  // the bf16 matmul output
                if (p.scale != 1.0f) s = bf16_round(s * p.scale);
                if (p.bias != nullptr && i < L && j < L)
                    s = bf16_round(s + __bfloat162float(p.bias[((long long)h * L + i) * L + j]));
                if (j >= L || (p.causal && j > i)) s = -INFINITY;
                sS[(rg + r) * Lp + j] = s;
            }
        }
    }
    __syncthreads();                                             // K fully consumed, scores complete
    // ---- stage V over K ----
    for (int i0 = tid; i0 < pieces; i0 += 8 * kSaThreads) {
        uint4 buf[8];
#pragma unroll
        for (int u = 0; u < 8; ++u) {
            const int i = i0 + u * kSaThreads, j = i >> 3, c = i & 7;
            buf[u] = (i < pieces && j < L) ? *reinterpret_cast<const uint4*>(p.v + (base + j) * p.ld + h * 64 + c * 8) : make_uint4(0, 0, 0, 0);
        }
#pragma unroll
        for (int u = 0; u < 8; ++u) {
            const int i = i0 + u * kSaThreads;
            if (i < pieces) *reinterpret_cast<uint4*>(sKV + (size_t)i * 8) = buf[u];          // [Lp][64]: piece i at element 8 i
        }
    }
    // ---- phase 2: softmax (warp w: rows 4w .. 4w+3) ----
    {
        const int warp = tid >> 5, lane = tid & 31;
        for (int r = warp * 4; r < warp * 4 + 4; ++r) {
            float m = -INFINITY;
            for (int j = lane; j < Lp; j += 32) m = fmaxf(m, sS[r * Lp + j]);
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
            float sum = 0.f;
            for (int j = lane; j < Lp; j += 32) {
                const float e = __expf(sS[r * Lp + j] - m);
                sS[r * Lp + j] = e;
                sum += e;
            }
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
            const float inv = 1.0f / sum;
            for (int j = lane; j < Lp; j += 32) sP[r * Lp + j] = __float2bfloat16_rn(sS[r * Lp + j] * inv);
        }
    }
    __syncthreads();
    // ---- phase 3: out = P V ----
    {
        const int r = tid >> 3, d0 = (tid & 7) * 8;
        float o[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
#pragma unroll 4
        for (int j = 0; j < L; ++j) {
            const float pj = __bfloat162float(sP[r * Lp + j]);
            const uint4 vv = *reinterpret_cast<const uint4*>(sKV + (size_t)j * 64 + d0);
            const uint32_t w[4] = {vv.x, vv.y, vv.z, vv.w};
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const float2 f = unpack_bf16x2(w[e]);
                o[2 * e] = fmaf(pj, f.x, o[2 * e]);
                o[2 * e + 1] = fmaf(pj, f.y, o[2 * e + 1]);
            }
        }
        if (row0 + r < L) {
            uint4 u;
            u.x = pack_bf16x2(o[0], o[1]); u.y = pack_bf16x2(o[2], o[3]); u.z = pack_bf16x2(o[4], o[5]); u.w = pack_bf16x2(o[6], o[7]);
            *reinterpret_cast<uint4*>(p.out + (base + row0 + r) * p.ldo + h * 64 + d0) = u;
        }
    }
}

}  // namespace vcb
