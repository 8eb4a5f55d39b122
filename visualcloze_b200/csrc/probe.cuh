// probe.cuh -- single-tile wgmma with caller-chosen operand descriptors (test hook, see vcb200.h).
// Pins the layout assumptions of gemm_sm90.cuh / attn_sm90.cuh on real hardware: K-major SW128 operands,
// MN-major SW128 B operand (the V tile of attention) and the bf16 A operand held in registers (the P tile).
#pragma once
#include "wgmma_sm90.cuh"

namespace vcb {

struct ProbeParams {
    const __nv_bfloat16* a;   // [128, K] row-major (used by the a_from_regs path)
    float* out;               // [128, 128]
    int ksteps;               // K = 16 * ksteps, 1..8
    int b_mn_major;
    int a_from_regs;
    uint32_t b_lbo, b_sbo, b_kstep_bytes;
};

// warps 0..7: two warpgroups, 64 rows each; warp 8: TMA
__global__ void __launch_bounds__(288, 1)
wgmma_probe_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b, const ProbeParams p) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint8_t* smem_a = smem;                 // 32 KB: two [128 x 64] K blocks
    uint8_t* smem_b = smem + 32768;         // 32 KB
    uint64_t* full = reinterpret_cast<uint64_t*>(smem + 65536);
    const uint32_t warp = warp_id_uniform(), lane = lane_id();
    const int K = 16 * p.ksteps;

    if (warp == 8 && lane == 0) {
        mbar_init(full, 1);
        fence_barrier_init();
    }
    __syncthreads();

    if (warp == 8) {
        if (lane == 0) {
            const int kblocks = (K + 63) / 64;
            // A: [128 rows, 64 cols] boxes; B: K-major -> same as A; MN-major -> two [K rows, 64 cols] boxes
            mbar_expect_tx(full, (uint32_t)(kblocks * 128 * 128 + (p.b_mn_major ? 2 * K * 128 : kblocks * 128 * 128)));
            for (int kb = 0; kb < kblocks; ++kb) tma_load_2d(&tmap_a, full, smem_a + kb * 16384, kb * 64, 0, kEvictNormal);
            if (p.b_mn_major) {
                tma_load_2d(&tmap_b, full, smem_b, 0, 0, kEvictNormal);
                tma_load_2d(&tmap_b, full, smem_b + K * 128, 64, 0, kEvictNormal);
            } else {
                for (int kb = 0; kb < kblocks; ++kb) tma_load_2d(&tmap_b, full, smem_b + kb * 16384, kb * 64, 0, kEvictNormal);
            }
        }
        return;
    }
    const int wg = (int)warp >> 2;
    const uint32_t q = lane & 3;
    const int row = wg * 64 + (int)(warp & 3) * 16 + (int)(lane >> 2);       // + 8 h
    float d[64];
    mbar_wait(full, 0);
    wgmma_fence();
    for (int ks = 0; ks < p.ksteps; ++ks) {
        const uint32_t a_off = (ks >> 2) * 16384 + (ks & 3) * 32;
        const uint64_t bdesc = p.b_mn_major ? make_smem_desc(smem_u32(smem_b) + ks * p.b_kstep_bytes, p.b_lbo, p.b_sbo)
                                            : make_smem_desc(smem_u32(smem_b) + a_off, 16, 1024);
        if (p.a_from_regs) {
            // A[row + 8 h, 16 ks + 8 i + 2 q .. + 1] as packed bf16 pairs, the accumulator's row layout
            uint32_t a[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) a[i] = *reinterpret_cast<const uint32_t*>(p.a + (row + 8 * (i & 1)) * K + 16 * ks + 8 * (i >> 1) + 2 * q);
            if (p.b_mn_major) wgmma_rs<128, true>(d, a, bdesc, ks != 0);
            else wgmma_rs<128, false>(d, a, bdesc, ks != 0);
        } else {
            const uint64_t adesc = make_smem_desc(smem_u32(smem_a) + wg * 64 * 128 + a_off, 16, 1024);
            if (p.b_mn_major) wgmma_ss<128, false, true>(d, adesc, bdesc, ks != 0);
            else wgmma_ss<128>(d, adesc, bdesc, ks != 0);
        }
    }
    wgmma_commit();
    wgmma_wait<0>();
#pragma unroll
    for (int i = 0; i < 64; ++i) p.out[(row + 8 * ((i >> 1) & 1)) * 128 + 8 * (i >> 2) + 2 * q + (i & 1)] = d[i];
}

}  // namespace vcb
