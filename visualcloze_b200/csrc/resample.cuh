// resample.cuh -- grid-cell preparation on the device: Pillow's 8-bit separable resampler (Image.resize on an RGB image,
// LANCZOS / BICUBIC, reducing_gap=None) and image_transform's ToTensor + Normalize(0.5, 0.5), bit-exact to both.
//
// One resample launch is one pass of Pillow's ImagingResample along one axis over an interleaved uint8 image [rows][cols][3]:
// output sample i of the pass reads the n = bounds[i][1] inputs starting at bounds[i][0] along that axis and forms
//     clamp((2^21 + sum_k coeffs[i][k] * in[xmin + k]) >> 22, 0, 255)
// in int32, exactly Pillow's ImagingResampleHorizontal_8bpc / ImagingResampleVertical_8bpc (the int32 weights are its
// normalize_coeffs_8bpc, built on the host by visualcloze_b200/resample.py).  A resize is a horizontal pass then a vertical one
// with a uint8 image in between; a pass whose axis keeps its size is skipped by the caller, as Pillow skips it.
// HBM / latency bound: one thread per output pixel, 3 channels, the window walked along the axis.
#pragma once
#include "vcb_common.cuh"

namespace vcb {

constexpr int kResamplePrecisionBits = 32 - 8 - 2;     // Pillow's PRECISION_BITS

VCB_DEVICE uint8_t resample_clip8(int acc) {
    const int v = acc >> kResamplePrecisionBits;
    return (uint8_t)(v < 0 ? 0 : (v > 255 ? 255 : v));
}

// kAxis 0: along x, out [in_h][out_n][3];  kAxis 1: along y, out [out_n][in_w][3].  Row strides in bytes.
// A window is clipped to [0, in_len) and to ksize taps, so no table can make the kernel read outside the input; the tables
// resample.py builds never need the clip.
template <int kAxis>
__global__ void resample_u8_kernel(const uint8_t* __restrict__ in, long long in_ld, int in_w, int in_h,
                                   const int* __restrict__ bounds, const int* __restrict__ coeffs, int ksize, int out_n,
                                   uint8_t* __restrict__ out, long long out_ld) {
    const int out_w = kAxis == 0 ? out_n : in_w;
    const int out_h = kAxis == 0 ? in_h : out_n;
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (long long)out_w * out_h) return;
    const int x = (int)(idx % out_w), y = (int)(idx / out_w);
    const int i = kAxis == 0 ? x : y;                                  // output sample along the axis
    const int in_len = kAxis == 0 ? in_w : in_h;
    int xmin = __ldg(bounds + 2 * i), n = __ldg(bounds + 2 * i + 1);
    const int* k = coeffs + (long long)i * ksize;
    int k0 = 0;
    if (xmin < 0) { k0 = -xmin; xmin = 0; }
    n = min(min(n, ksize) - k0, in_len - xmin);
    const long long step = kAxis == 0 ? 3 : in_ld;
    const uint8_t* p = kAxis == 0 ? in + (long long)y * in_ld + 3LL * xmin : in + (long long)xmin * in_ld + 3LL * x;
    int s0 = 1 << (kResamplePrecisionBits - 1), s1 = s0, s2 = s0;
    for (int t = 0; t < n; ++t, p += step) {
        const int w = __ldg(k + k0 + t);
        s0 += (int)p[0] * w;
        s1 += (int)p[1] * w;
        s2 += (int)p[2] * w;
    }
    uint8_t* o = out + (long long)y * out_ld + 3LL * x;
    o[0] = resample_clip8(s0);
    o[1] = resample_clip8(s1);
    o[2] = resample_clip8(s2);
}

// A crop box of a uint8 image [in_h][in_w][3] -> fp32 planes out[c][y][col0 + x] = (u / 255 - 0.5) / 0.5, each operation
// rounded as torch's fp32 true division and subtraction round it (image_transform).  Box pixels outside the image read 0
// (Pillow's crop pads with zeros) and become -1; an empty image (in_w or in_h 0) is a blank cell.
__global__ void cell_to_model_input_kernel(const uint8_t* __restrict__ in, long long in_ld, int in_w, int in_h, int crop_x,
                                           int crop_y, int crop_w, int crop_h, float* __restrict__ out, long long ld_row,
                                           long long ld_plane, int col0) {
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (long long)crop_w * crop_h) return;
    const int x = (int)(idx % crop_w), y = (int)(idx / crop_w);
    const int sx = crop_x + x, sy = crop_y + y;
    const bool inside = sx >= 0 && sx < in_w && sy >= 0 && sy < in_h;
    const uint8_t* p = in + (long long)sy * in_ld + 3LL * sx;
    float* o = out + (long long)y * ld_row + col0 + x;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        const float u = inside ? (float)p[c] : 0.f;
        o[c * ld_plane] = __fdiv_rn(__fsub_rn(__fdiv_rn(u, 255.f), 0.5f), 0.5f);
    }
}

}  // namespace vcb
