// host_util.cuh -- host-side plumbing shared by the C-ABI translation units: error string, launch counter,
// device checks, and TMA tensor-map construction through the driver entry point (no link-time libcuda dependency).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>

#include <atomic>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <mutex>
#include <vector>

namespace vcb {

inline char* error_buf() {
    static thread_local char buf[512] = {0};
    return buf;
}
inline int set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(error_buf(), 512, fmt, ap);
    va_end(ap);
    return 1;
}
inline std::atomic<long long>& launch_counter() {
    static std::atomic<long long> c{0};
    return c;
}
inline void count_launch() { launch_counter().fetch_add(1, std::memory_order_relaxed); }

inline int check_launch(const char* what) {
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return set_error("%s launch failed: %s", what, cudaGetErrorString(e));
    count_launch();
    return 0;
}

// ---- optional per-category device timing (bench.py roofline numbers): CUDA events around every launch ------------
enum ProfCat : int { PROF_GEMM = 0, PROF_ATTN = 1, PROF_LN = 2, PROF_OTHER = 3, PROF_CONV = 4, PROF_VAE_EW = 5, PROF_NCAT = 6 };
// info: what was launched -- GEMM {M, N, K, epilogue | (block_n / 32) << 8 | cta_group << 16 | VAE context << 24}, conv {pixels, cout, 9 cin, stride},
// attention {B, L, heads, fixed-reference softmax | persistent << 1}, others zero
struct ProfRec { int cat; cudaEvent_t a, b; int info[4]; };
struct Profiler {
    bool on = false;
    std::vector<ProfRec> recs;
    std::vector<cudaEvent_t> pool;
    cudaEvent_t get() {
        if (!pool.empty()) { cudaEvent_t e = pool.back(); pool.pop_back(); return e; }
        cudaEvent_t e;
        cudaEventCreate(&e);
        return e;
    }
};
inline Profiler& profiler() {
    static Profiler p;
    return p;
}
// launches issued from inside the VAE engine are marked (bit 24 of a GEMM record's info[3]): the decoder's 1x1 convolutions and
// mid-block attention products run on the same GEMM entry point as the FLUX-DiT's Linears
inline int& prof_context() {
    static thread_local int c = 0;
    return c;
}
struct ProfContext {
    int prev;
    explicit ProfContext(int c) : prev(prof_context()) { prof_context() = c; }
    ~ProfContext() { prof_context() = prev; }
};
struct ProfScope {
    cudaStream_t st;
    cudaEvent_t b = nullptr;
    size_t idx = 0;
    ProfScope(int cat, void* stream, int i0 = 0, int i1 = 0, int i2 = 0, int i3 = 0) : st((cudaStream_t)stream) {
        Profiler& p = profiler();
        if (!p.on) return;
        cudaEvent_t a = p.get();
        b = p.get();
        cudaEventRecord(a, st);
        idx = p.recs.size();
        p.recs.push_back({cat, a, b, {i0, i1, i2, cat == PROF_GEMM ? (i3 | (prof_context() << 24)) : i3}});
    }
    void set_info(int k, int v) {
        if (b) profiler().recs[idx].info[k] = v;
    }
    ~ProfScope() {
        if (b) cudaEventRecord(b, st);
    }
};

// launch with programmatic stream serialization (the kernel must execute griddepcontrol.wait before touching inputs)
template <class Kern, class... Args>
inline cudaError_t launch_pdl(Kern kern, dim3 grid, dim3 block, size_t smem, cudaStream_t st, int cluster_x, Args... args) {
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = st;
    cudaLaunchAttribute attr[2];
    int n = 0;
    static const bool pdl = [] { const char* e = getenv("VCB_NO_PDL"); return !(e && atoi(e)); }();
    if (pdl) {
        attr[n].id = cudaLaunchAttributeProgrammaticStreamSerialization;
        attr[n].val.programmaticStreamSerializationAllowed = 1;
        ++n;
    }
    if (cluster_x > 1) {
        attr[n].id = cudaLaunchAttributeClusterDimension;
        attr[n].val.clusterDim.x = cluster_x;
        attr[n].val.clusterDim.y = 1;
        attr[n].val.clusterDim.z = 1;
        ++n;
    }
    cfg.attrs = attr;
    cfg.numAttrs = n;
    return cudaLaunchKernelEx(&cfg, kern, args...);
}

struct DeviceInfo {
    int ok = 0;
    int sms = 0;
    int cc_major = 0, cc_minor = 0;
    char err[256] = {0};
};
inline DeviceInfo& device_info() {
    static DeviceInfo info;
    static std::once_flag once;
    std::call_once(once, [] {
        int dev = 0;
        cudaError_t e = cudaGetDevice(&dev);
        if (e != cudaSuccess) {
            snprintf(info.err, sizeof(info.err), "no CUDA device: %s (libvcb200 has no CPU fallback)", cudaGetErrorString(e));
            return;
        }
        cudaDeviceGetAttribute(&info.sms, cudaDevAttrMultiProcessorCount, dev);
        cudaDeviceGetAttribute(&info.cc_major, cudaDevAttrComputeCapabilityMajor, dev);
        cudaDeviceGetAttribute(&info.cc_minor, cudaDevAttrComputeCapabilityMinor, dev);
        if (info.cc_major != 9) {
            snprintf(info.err, sizeof(info.err), "device is sm_%d%d; libvcb200 is built for sm_90a only", info.cc_major, info.cc_minor);
            return;
        }
        info.ok = 1;
    });
    return info;
}
inline int ensure_device() {
    DeviceInfo& d = device_info();
    if (!d.ok) return set_error("%s", d.err);
    return 0;
}
inline int num_sms() { return device_info().sms; }

// ---- TMA tensor maps ---------------------------------------------------------------------------
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
inline PFN_encodeTiled encode_fn() {
    static PFN_encodeTiled fn = [] {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q);
        if (e != cudaSuccess || q != cudaDriverEntryPointSuccess) return (PFN_encodeTiled) nullptr;
        return (PFN_encodeTiled)p;
    }();
    return fn;
}

// bf16 tensor, dims given innermost-first; strides in ELEMENTS for dims 1.. ; 128-byte swizzle; OOB reads give zeros
// elem_bytes: 2 = bf16 (default), 1 = 8-bit (e4m3 operands of the fp8 GEMM)
inline int make_tmap(CUtensorMap* m, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_elems,
                     const uint32_t* box, const uint32_t* elem_strides = nullptr, int elem_bytes = 2) {
    PFN_encodeTiled fn = encode_fn();
    if (!fn) return set_error("cuTensorMapEncodeTiled entry point not available");
    if ((reinterpret_cast<uintptr_t>(base) & 15) != 0) return set_error("TMA base pointer must be 16-byte aligned");
    cuuint64_t gdims[5];
    cuuint64_t gstr[4];
    cuuint32_t gbox[5], estr[5];
    for (int i = 0; i < rank; ++i) {
        gdims[i] = dims[i];
        gbox[i] = box[i];
        estr[i] = elem_strides ? elem_strides[i] : 1;
        if (i > 0) {
            gstr[i - 1] = strides_elems[i - 1] * (uint64_t)elem_bytes;
            if (gstr[i - 1] % 16) return set_error("TMA stride must be a multiple of 16 bytes");
        }
    }
    if (box[0] * (uint32_t)elem_bytes > 128) return set_error("TMA inner box exceeds the 128-byte swizzle span");
    CUresult r = fn(m, elem_bytes == 1 ? CU_TENSOR_MAP_DATA_TYPE_UINT8 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, (cuuint32_t)rank, const_cast<void*>(base), gdims, gstr, gbox, estr,
                    CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                    CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return set_error("cuTensorMapEncodeTiled failed with CUresult %d", (int)r);
    return 0;
}
inline int make_tmap_2d(CUtensorMap* m, const void* base, uint64_t cols, uint64_t rows, uint64_t ld, uint32_t box_cols,
                        uint32_t box_rows, int elem_bytes = 2) {
    const uint64_t dims[2] = {cols, rows};
    const uint64_t str[1] = {ld};
    const uint32_t box[2] = {box_cols, box_rows};
    return make_tmap(m, base, 2, dims, str, box, nullptr, elem_bytes);
}
inline int make_tmap_3d(CUtensorMap* m, const void* base, uint64_t cols, uint64_t rows, uint64_t batch, uint64_t ld,
                        uint64_t batch_stride, uint32_t box_cols, uint32_t box_rows, int elem_bytes = 2) {
    const uint64_t dims[3] = {cols, rows, batch};
    const uint64_t str[2] = {ld, batch_stride};
    const uint32_t box[3] = {box_cols, box_rows, 1};
    return make_tmap(m, base, 3, dims, str, box, nullptr, elem_bytes);
}
inline int make_tmap_4d(CUtensorMap* m, const void* base, const uint64_t dims[4], const uint64_t strides_elems[3],
                        const uint32_t box[4], const uint32_t* elem_strides = nullptr) {
    return make_tmap(m, base, 4, dims, strides_elems, box, elem_strides);
}

}  // namespace vcb
