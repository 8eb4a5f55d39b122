// vae_kernels.cuh -- HBM-bound kernels of the VAE decoder (models/modules/autoencoder.py): GroupNorm(32)+swish,
// nearest 2x upsampling, row softmax of the mid-block attention, latent-token / image layout conversions.
// Activations are NHWC bf16 so that a pixel's channels are one contiguous, 16-byte-vectorisable run and the 3x3
// convolutions are implicit GEMMs (gemm_sm90.cuh, A_CONV3X3).
#pragma once
#include "vcb_common.cuh"

namespace vcb {

constexpr int kGnGroups = 32;
constexpr int kGnThreads = 256;
constexpr int kGnPixelsPerBlock = 256;

// ---- GroupNorm statistics, pass 1: per (image, pixel-chunk) partial (sum, sumsq) of every group -------------------
// x [n, P, C] bf16; part [n, chunks, 32, 2] fp32.  Thread layout: (pixel lane, channel pair); a warp reads
// consecutive channel pairs of one pixel (coalesced).  Deterministic: no atomics.
__global__ void __launch_bounds__(kGnThreads)
gn_partial_kernel(const __nv_bfloat16* __restrict__ x, float* __restrict__ part, int P, int C) {
    const int n = blockIdx.y, chunk = blockIdx.x;
    const int pairs = C >> 1;                         // channel pairs per pixel (C <= 512, C % 32 == 0)
    const int lanes = kGnThreads / pairs;             // pixels processed concurrently (>= 1 since pairs <= 256)
    const int cp = threadIdx.x % pairs, pl = threadIdx.x / pairs;
    const int p0 = chunk * kGnPixelsPerBlock;
    const int p1 = min(P, p0 + kGnPixelsPerBlock);
    float s0 = 0.f, q0 = 0.f, s1 = 0.f, q1 = 0.f;
    if (pl < lanes) {
        const __nv_bfloat16* base = x + ((long long)n * P) * C + 2 * cp;
        for (int p = p0 + pl; p < p1; p += lanes) {
            float2 f = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(base + (long long)p * C));
            s0 += f.x; q0 = fmaf(f.x, f.x, q0);
            s1 += f.y; q1 = fmaf(f.y, f.y, q1);
        }
    }
    // per-channel partials [lane][channel]; lanes * C == 2 * kGnThreads floats
    __shared__ float sh_s[2 * kGnThreads], sh_q[2 * kGnThreads];
    if (pl < lanes) {
        sh_s[pl * C + 2 * cp] = s0; sh_s[pl * C + 2 * cp + 1] = s1;
        sh_q[pl * C + 2 * cp] = q0; sh_q[pl * C + 2 * cp + 1] = q1;
    }
    __syncthreads();
    if (threadIdx.x < kGnGroups) {
        const int g = threadIdx.x;
        const int cpg = C / kGnGroups;                // channels per group
        float ts = 0.f, tq = 0.f;
        for (int l = 0; l < lanes; ++l)
            for (int c = 0; c < cpg; ++c) {
                ts += sh_s[l * C + g * cpg + c];
                tq += sh_q[l * C + g * cpg + c];
            }
        float* o = part + (((long long)n * gridDim.x + chunk) * kGnGroups + g) * 2;
        o[0] = ts;
        o[1] = tq;
    }
}

// pass 2: stats[n, 32] = (mean, rstd), eps 1e-6; one warp per (n, group)
__global__ void gn_finalize_kernel(const float* __restrict__ part, float2* __restrict__ stats, int chunks, long long count) {
    const int n = blockIdx.y, g = blockIdx.x, lane = threadIdx.x;
    float s = 0.f, q = 0.f;
    for (int c = lane; c < chunks; c += 32) {
        const float* pp = part + (((long long)n * chunks + c) * kGnGroups + g) * 2;
        s += pp[0];
        q += pp[1];
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        s += __shfl_xor_sync(0xffffffffu, s, o);
        q += __shfl_xor_sync(0xffffffffu, q, o);
    }
    if (lane == 0) {
        const float mean = s / (float)count;
        const float var = fmaxf(q / (float)count - mean * mean, 0.f);
        stats[n * kGnGroups + g] = make_float2(mean, rsqrtf(var + 1e-6f));
    }
}

// pass 3: y = swish((x - mean) * rstd * gamma + beta) (or without swish), bf16 out; 8 channels per thread
__global__ void gn_apply_kernel(const __nv_bfloat16* __restrict__ x, __nv_bfloat16* __restrict__ y,
                                const float2* __restrict__ stats, const float* __restrict__ gamma,
                                const float* __restrict__ beta, long long P, int C, int swish) {
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;     // over n * P * C / 8
    const int c8 = C >> 3;
    const long long total = (long long)gridDim.y * P * c8;
    (void)total;
    const int n = blockIdx.y;
    if (idx >= P * c8) return;
    const int c0 = (int)(idx % c8) * 8;
    const long long off = ((long long)n * P) * C + idx * 8;
    const float2 st = stats[n * kGnGroups + c0 / (C / kGnGroups)];               // 8 | C/32 or C/32 == 4 -> see host check
    uint4 u = *reinterpret_cast<const uint4*>(x + off);
    const uint32_t w[4] = {u.x, u.y, u.z, u.w};
    uint32_t o[4];
    const int cpg = C / kGnGroups;
#pragma unroll
    for (int e = 0; e < 4; ++e) {
        float2 f = unpack_bf16x2(w[e]);
        const int ca = c0 + 2 * e, cb = ca + 1;
        const float2 sa = cpg >= 8 ? st : stats[n * kGnGroups + ca / cpg];
        const float2 sb = cpg >= 8 ? st : stats[n * kGnGroups + cb / cpg];
        float va = (f.x - sa.x) * sa.y * __ldg(gamma + ca) + __ldg(beta + ca);
        float vb = (f.y - sb.x) * sb.y * __ldg(gamma + cb) + __ldg(beta + cb);
        if (swish) {
            va = va / (1.0f + __expf(-va));
            vb = vb / (1.0f + __expf(-vb));
        }
        o[e] = pack_bf16x2(va, vb);
    }
    *reinterpret_cast<uint4*>(y + off) = make_uint4(o[0], o[1], o[2], o[3]);
}

// nearest-neighbour 2x upsampling, NHWC: out[n, y, x, :] = in[n, y/2, x/2, :]   (autoencoder.py:104)
__global__ void upsample2x_kernel(const __nv_bfloat16* __restrict__ in, __nv_bfloat16* __restrict__ out, int H, int W, int C) {
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;     // over (2H)(2W)(C/8)
    const int c8 = C >> 3, n = blockIdx.y;
    const long long per = (long long)(2 * H) * (2 * W) * c8;
    if (idx >= per) return;
    const int c = (int)(idx % c8);
    const long long pix = idx / c8;
    const int ox = (int)(pix % (2 * W)), oy = (int)(pix / (2 * W));
    const uint4 v = *reinterpret_cast<const uint4*>(in + (((long long)n * H + (oy >> 1)) * W + (ox >> 1)) * C + c * 8);
    *reinterpret_cast<uint4*>(out + ((long long)n * per + idx) * 8) = v;
}

// row softmax of fp32 scores: p[r, :] = bf16(softmax(scale * s[r, :]))   (single-head attention of AttnBlock)
__global__ void __launch_bounds__(256)
softmax_rows_kernel(const float* __restrict__ s, __nv_bfloat16* __restrict__ p, int cols, long long lds, long long ldp, float scale) {
    const long long r = blockIdx.x;
    const float* sr = s + r * lds;
    __shared__ float red[8];
    float m = -INFINITY;
    for (int c = threadIdx.x; c < cols; c += 256) m = fmaxf(m, sr[c]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
    __syncthreads();
    m = red[0];
#pragma unroll
    for (int i = 1; i < 8; ++i) m = fmaxf(m, red[i]);
    __syncthreads();
    float sum = 0.f;
    for (int c = threadIdx.x; c < cols; c += 256) sum += __expf((sr[c] - m) * scale);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = sum;
    __syncthreads();
    sum = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) sum += red[i];
    const float inv = 1.0f / sum;
    __nv_bfloat16* pr = p + r * ldp;
    for (int c = threadIdx.x; c < cols; c += 256) pr[c] = __float2bfloat16_rn(__expf((sr[c] - m) * scale) * inv);
}

// packed latent tokens [n, h*w, 4*zc] ("(h w) (c ph pw)", visualcloze.py:428) -> NHWC [n, 2h, 2w, cpad] with
// z / scale_factor + shift_factor applied in bf16 steps (visualcloze.py:430), channels >= zc zero
__global__ void tokens_to_nhwc_kernel(const __nv_bfloat16* __restrict__ tok, __nv_bfloat16* __restrict__ out, int h, int w,
                                      int zc, int cpad, float scale_factor, float shift_factor) {
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;     // over (2h)(2w)(cpad)
    const int n = blockIdx.y;
    const long long per = (long long)(2 * h) * (2 * w) * cpad;
    if (idx >= per) return;
    const int c = (int)(idx % cpad);
    const long long pix = idx / cpad;
    const int x = (int)(pix % (2 * w)), y = (int)(pix / (2 * w));
    float v = 0.f;
    if (c < zc) {
        const int t = (y >> 1) * w + (x >> 1);
        const int d = c * 4 + (y & 1) * 2 + (x & 1);
        const float z = __bfloat162float(tok[((long long)n * h * w + t) * (4 * zc) + d]);
        v = bf16_round(bf16_round(z / scale_factor) + shift_factor);
    }
    out[(long long)n * per + idx] = __float2bfloat16_rn(v);
}

// decoder output NHWC [n, H, W, cpad] -> fp32 CHW [n, 3, H, W] (raw) and/or uint8 CHW image:
// (x + 1) / 2 -> clamp(0, 1) in bf16 steps (visualcloze.py:431-432), then float * 255 truncated (to_pil_image)
__global__ void nhwc_to_image_kernel(const __nv_bfloat16* __restrict__ in, float* __restrict__ raw, uint8_t* __restrict__ img,
                                     int H, int W, int cpad, int out_ch) {
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;     // over out_ch * H * W
    const int n = blockIdx.y;
    const long long per = (long long)out_ch * H * W;
    if (idx >= per) return;
    const int c = (int)(idx / ((long long)H * W));
    const long long pix = idx % ((long long)H * W);
    const float v = __bfloat162float(in[((long long)n * H * W + pix) * cpad + c]);
    if (raw) raw[(long long)n * per + idx] = v;
    if (img) {
        float t = bf16_round(bf16_round(v + 1.0f) / 2.0f);
        t = fminf(fmaxf(t, 0.f), 1.f);
        img[(long long)n * per + idx] = (uint8_t)(t * 255.0f);
    }
}

// image [n, cin, H, W] fp32 (NCHW, values in [-1, 1]) -> NHWC bf16 [n, H, W, cpad], channels >= cin zero (encoder input)
__global__ void image_to_nhwc_kernel(const float* __restrict__ img, __nv_bfloat16* __restrict__ out, int H, int W, int cin, int cpad) {
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;     // over H * W * cpad
    const int n = blockIdx.y;
    const long long per = (long long)H * W * cpad;
    if (idx >= per) return;
    const int c = (int)(idx % cpad);
    const long long pix = idx / cpad;
    float v = 0.f;
    if (c < cin) v = img[((long long)n * cin + c) * H * W + pix];
    out[(long long)n * per + idx] = __float2bfloat16_rn(v);
}

// encoder output moments NHWC [n, h2, w2, 2*zc] bf16 (mean | logvar) -> latent sample mean + exp(0.5 logvar) * noise
// (DiagonalGaussian, autoencoder.py:262-275; bf16 steps) -> (z - shift) * scale (visualcloze.py:378) -> packed tokens
// [n, (h2/2)(w2/2), 4*zc] ("c (h 2)(w 2) -> (h w)(c 2 2)", visualcloze.py:385).  noise [n, zc, h2, w2] fp32 or NULL (mode).
// Optionally also writes the raw moments as fp32 NCHW [n, 2*zc, h2, w2].
__global__ void moments_to_tokens_kernel(const __nv_bfloat16* __restrict__ mom, const float* __restrict__ noise,
                                         __nv_bfloat16* __restrict__ tok, float* __restrict__ raw, int h2, int w2, int zc,
                                         float scale_factor, float shift_factor) {
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;     // over h2 * w2 * zc
    const int n = blockIdx.y;
    const long long per = (long long)h2 * w2 * zc;
    if (idx >= per) return;
    const int c = (int)(idx % zc);
    const long long pix = idx / zc;
    const int x = (int)(pix % w2), y = (int)(pix / w2);
    const __nv_bfloat16* m = mom + ((long long)n * h2 * w2 + pix) * (2 * zc);
    const float mean = __bfloat162float(m[c]), logvar = __bfloat162float(m[zc + c]);
    if (raw) {
        raw[(((long long)n * 2 * zc + c) * h2 + y) * w2 + x] = mean;
        raw[(((long long)n * 2 * zc + zc + c) * h2 + y) * w2 + x] = logvar;
    }
    float z = mean;
    if (noise) {
        const float stdv = bf16_round(expf(bf16_round(0.5f * logvar)));
        const float eps = bf16_round(noise[(((long long)n * zc + c) * h2 + y) * w2 + x]);
        z = bf16_round(mean + bf16_round(stdv * eps));
    }
    z = bf16_round(bf16_round(z - shift_factor) * scale_factor);
    const int w = w2 >> 1;
    const long long t = (long long)(y >> 1) * w + (x >> 1);
    tok[((long long)n * (h2 >> 1) * w + t) * (4 * zc) + c * 4 + (y & 1) * 2 + (x & 1)] = __float2bfloat16_rn(z);
}

}  // namespace vcb
