// vcb_common.cuh -- sm_90a PTX wrappers shared by the vcb200 kernels (mbarrier, TMA, wgmma operand descriptors).
// Hand-written inline PTX; bit layouts follow the PTX ISA "wgmma" matrix descriptor.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace vcb {

#define VCB_DEVICE __device__ __forceinline__

// ------------------------------------------------------------------------------------------
// misc
// ------------------------------------------------------------------------------------------
VCB_DEVICE uint32_t smem_u32(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }
VCB_DEVICE uint32_t lane_id() { return threadIdx.x & 31; }
VCB_DEVICE uint32_t warp_id_uniform() { return __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0); }

VCB_DEVICE bool elect_one() {
    uint32_t pred;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "elect.sync _|p, 0xffffffff;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}\n"
        : "=r"(pred));
    return pred != 0;
}

VCB_DEVICE uint32_t cluster_ctarank() {
    uint32_t r;
    asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
    return r;
}
VCB_DEVICE void cluster_arrive() { asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory"); }
VCB_DEVICE void cluster_wait() { asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory"); }
VCB_DEVICE void cluster_sync() { cluster_arrive(); cluster_wait(); }

// bf16 helpers: round-to-nearest-even through the bf16 grid, staying in fp32
VCB_DEVICE float bf16_round(float x) { return __bfloat162float(__float2bfloat16_rn(x)); }
VCB_DEVICE uint32_t pack_bf16x2(float lo, float hi) {
    __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
    return *reinterpret_cast<uint32_t*>(&v);
}
VCB_DEVICE float2 unpack_bf16x2(uint32_t u) {
    __nv_bfloat162 v = *reinterpret_cast<__nv_bfloat162*>(&u);
    return __bfloat1622float2(v);
}

// ------------------------------------------------------------------------------------------
// mbarrier
// ------------------------------------------------------------------------------------------
VCB_DEVICE void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
VCB_DEVICE void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
VCB_DEVICE void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

VCB_DEVICE void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
                 : "memory");
}
VCB_DEVICE void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
// arrive on the barrier at the same smem offset in CTA `cta` of the cluster
VCB_DEVICE void mbar_arrive_cluster(uint64_t* bar, uint32_t cta) {
    uint32_t remote;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(remote) : "r"(smem_u32(bar)), "r"(cta));
    asm volatile("mbarrier.arrive.release.cluster.shared::cluster.b64 _, [%0];" ::"r"(remote) : "memory");
}
VCB_DEVICE bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}\n"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    return ok != 0;
}
VCB_DEVICE void mbar_wait(uint64_t* bar, uint32_t parity) {
    while (!mbar_try_wait(bar, parity)) {
    }
}

// ------------------------------------------------------------------------------------------
// TMA (cp.async.bulk.tensor)
// ------------------------------------------------------------------------------------------
constexpr uint64_t kEvictNormal = 0x1000000000000000ull;
constexpr uint64_t kEvictFirst = 0x12F0000000000000ull;
constexpr uint64_t kEvictLast = 0x14F0000000000000ull;

VCB_DEVICE void tma_prefetch_desc(const CUtensorMap* m) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}

// smem -> global tile store (bulk async-group completion); the destination may be peer memory mapped over NVLink
VCB_DEVICE void tma_store_2d(const CUtensorMap* m, const void* src_smem, int c0, int c1) {
    asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];" ::"l"(reinterpret_cast<uint64_t>(m)),
                 "r"(smem_u32(src_smem)), "r"(c0), "r"(c1)
                 : "memory");
}
VCB_DEVICE void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
VCB_DEVICE void tma_store_wait_read() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }   // smem reusable
VCB_DEVICE void tma_store_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }         // writes done

// kMulticast: the tile lands at the same shared-memory offset in every CTA of `mask` (a 2-CTA cluster sharing one B tile) and
// completes the transaction bytes on the barrier at the same offset in each of them.
template <bool kMulticast = false>
VCB_DEVICE void tma_load_2d(const CUtensorMap* m, uint64_t* bar, void* dst, int c0, int c1, uint64_t hint, uint16_t mask = 0) {
    if constexpr (kMulticast) {
        asm volatile(
            "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster.L2::cache_hint"
            " [%0], [%1, {%3, %4}], [%2], %5, %6;" ::"r"(smem_u32(dst)),
            "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "h"(mask), "l"(hint)
            : "memory");
    } else {
        asm volatile(
            "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint"
            " [%0], [%1, {%3, %4}], [%2], %5;" ::"r"(smem_u32(dst)),
            "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "l"(hint)
            : "memory");
    }
}
VCB_DEVICE void tma_load_3d(const CUtensorMap* m, uint64_t* bar, void* dst, int c0, int c1, int c2, uint64_t hint) {
    asm volatile(
        "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint"
        " [%0], [%1, {%3, %4, %5}], [%2], %6;" ::"r"(smem_u32(dst)),
        "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "l"(hint)
        : "memory");
}
VCB_DEVICE void tma_load_4d(const CUtensorMap* m, uint64_t* bar, void* dst, int c0, int c1, int c2, int c3, uint64_t hint) {
    asm volatile(
        "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint"
        " [%0], [%1, {%3, %4, %5, %6}], [%2], %7;" ::"r"(smem_u32(dst)),
        "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "l"(hint)
        : "memory");
}

// ------------------------------------------------------------------------------------------
// wgmma operands (the instruction wrappers are in wgmma_sm90.cuh)
// ------------------------------------------------------------------------------------------
// Shared-memory matrix descriptor (PTX ISA "Matrix descriptor" of wgmma):
//   [0,14) start address >> 4   [16,30) leading-dim byte offset >> 4   [32,46) stride-dim byte offset >> 4
//   [62,64) swizzle: 0 none, 1 = 128B, 2 = 64B, 3 = 32B
// K-major 128B-swizzled operand: rows of 128 bytes, SBO = 1024 (8 rows), LBO unused; a 16-element k step is +32 bytes.
// MN-major 128B-swizzled operand: LBO = distance between 64-element column blocks, SBO = 1024 (8 k rows).
VCB_DEVICE uint64_t make_smem_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
    uint64_t d = 0;
    d |= (uint64_t)((saddr & 0x3FFFFu) >> 4);
    d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFFu) << 16;
    d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFFu) << 32;
    d |= (uint64_t)1 << 62;                      // 128-byte swizzle
    return d;
}

// warp-specialised kernels hand the producer warpgroup's registers to the consumers (counts are multiples of 8)
template <int kRegs>
VCB_DEVICE void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(kRegs)); }
template <int kRegs>
VCB_DEVICE void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(kRegs)); }

VCB_DEVICE float ex2_approx(float x) {
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}

VCB_DEVICE int ld_acquire_gpu(const int* p) {
    int v;
    asm volatile("ld.acquire.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
VCB_DEVICE void st_release_gpu(int* p, int v) { asm volatile("st.release.gpu.global.s32 [%0], %1;" ::"l"(p), "r"(v) : "memory"); }

// Programmatic dependent launch: let the next kernel's CTAs start (and run their prologue) while this grid drains;
// `pdl_wait` blocks until the preceding grid has completed and its writes are visible.
VCB_DEVICE void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
VCB_DEVICE void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

// named barrier among `nthreads` threads (ids 1..15; 0 is __syncthreads)
VCB_DEVICE void named_bar_sync(uint32_t id, uint32_t nthreads) {
    asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

// activations (fp32 in/out)
VCB_DEVICE float gelu_tanh(float x) {
    // torch GELU(approximate="tanh"): 0.5 x (1 + tanh(sqrt(2/pi) (x + 0.044715 x^3)))
    // 0.5 (1 + tanh(u)) == sigmoid(2u): one ex2 + one fast divide instead of tanhf
    const float kBeta = 0.7978845608028654f, kKappa = 0.044715f;
    float inner = kBeta * (x + kKappa * x * x * x);
    return __fdividef(x, 1.0f + __expf(-2.0f * inner));
}
// the same function through tanh.approx.f32 (one MUFU, relative error 2^-11): the fp8 instantiations only -- their output is already
// off the reference's bf16 grid, and their epilogue, not the tensor pipe, bounds the short-K tiles
VCB_DEVICE float gelu_tanh_fast(float x) {
    const float kBeta = 0.7978845608028654f, kKappa = 0.044715f;
    const float u = x * fmaf(kBeta * kKappa, x * x, kBeta);
    float t;
    asm("tanh.approx.f32 %0, %1;" : "=f"(t) : "f"(u));
    const float hx = 0.5f * x;
    return fmaf(hx, t, hx);
}
VCB_DEVICE float silu(float x) { return x / (1.0f + __expf(-x)); }

}  // namespace vcb
