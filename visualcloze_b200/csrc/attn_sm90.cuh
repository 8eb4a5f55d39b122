// attn_sm90.cuh -- joint attention forward for sm_90a: wgmma, scores / probabilities / output in registers.
//
// Contract: attn_common.cuh (models/math.py:63-99; per-sample seqlens instead of unpad/pad).  One 128-query tile per unit of work:
//   warpgroup 0     TMA producer   Q once per segment; K/V tiles through a ring of 32 KB slots in the order K0 V0 K1 V1 ...
//   warpgroups 1,2  consumers      64 query rows each: S = Q K_j^T (wgmma, operands in smem) -> softmax in registers (a row lives in
//                                  the four lanes of a quad) -> O += P V_j (wgmma, P from registers, V MN-major in smem).  While one
//                                  warpgroup does its exponentials the tensor cores run the other's products.
// kFixed: a caller-promised bound of the scaled scores (QK-RMSNorm) replaces the running row max -- no max pass over S, no O
// rescaling (softmax is shift invariant; layers.py:63-84 bounds |q| and |k| by the norm scales).
//
// Two schedules share the kernel (AttnSkParams::ws == nullptr selects the first):
//   per-tile grid   one CTA per (query tile, head, sample); takes right-padded batches (seqlens) and the sequence-parallel routing.
//   persistent      grid = min(#SMs, ...) CTAs, equal contiguous shares of the (unit, key tile) space.  Full rounds of units are dealt
//                   out exactly like the per-tile grid (same L2 behaviour, no per-CTA prologue / drain between them); the units of
//                   the partial last round are cut along the key tiles into equal contiguous shares (see AttnSched).  A CTA's work
//                   is a sequence of SEGMENTS (unit, key tiles [kv0, kv1)):
//   * a segment covering all key tiles is finished locally (normalise, store);
//   * a unit cut by a share boundary is produced by several CTAs.  The piece holding key tile 0 -- always the LAST segment of its
//     CTA -- is the finaliser; every other piece -- always the FIRST phase-2 segment of its CTA, which waits on nothing -- dumps its
//     un-normalised (O, l[, m]) to its workspace slot and raises its flag.  The finaliser folds them in its epilogue:
//         fixed-reference softmax:  O = sum O_i, l = sum l_i            (all pieces share the reference exponent)
//         online max:               m = max m_i, O = sum O_i 2^(m_i - m), l likewise
//     Waiters only wait on CTAs with a larger index whose contribution is their first piece: deadlock-free with all CTAs
//     co-resident (grid <= #SMs, one CTA per SM).  Spin loops carry a watchdog that traps instead of hanging the GPU.
#pragma once
#include "attn_common.cuh"
#include "wgmma_sm90.cuh"

namespace vcb {

constexpr int kAttnThreads = 384;           // producer warpgroup + 2 consumer warpgroups
constexpr int kAttnConsumers = 256;
constexpr int kAttnSlots = 4;               // K/V ring of 32 KB slots
constexpr int kAttn4MaxSegs = 64;           // segments per CTA (the host uses the per-tile grid beyond that)
constexpr int kAttnSmemBytes = (1 + kAttnSlots) * kSlotBytes + 1024 + 256 + kAttn4MaxSegs * 32;
constexpr int kAttn4SlotFloats = 128 * 128 + 128 + 128;   // O [64 registers][256 threads] | l [128] | m [128]

struct AttnSkParams {
    float* ws;          // [gridDim.x][kAttn4SlotFloats]; null = per-tile grid
    int* flags;         // [gridDim.x]
    int epoch;          // value that marks "this launch's partial is ready"
    int no_split;       // experiment switch: deal the units of the partial last round out whole (no key-tile split, no partials)
    unsigned long long* timeline;   // optional [gridDim.x][kAttn4MaxSegs + 2] globaltimer stamps: start, end of every segment (debug)
};

// Schedule.  Units (sample, head, query tile) in that order; n_units = samples * heads * tiles.
//   phase 1  the R = n_units / G full rounds exactly like the per-tile grid: round r gives unit r * G + c to CTA c, so the CTAs
//            that run concurrently stream the same few heads' K / V through L2 (split only the tail, like the GEMM's stream-K).
//   phase 2  the rem = n_units % G units of the partial last round are cut along the key tiles into G2 equal contiguous ranges of the
//            flattened (unit, key tile) space, one per CTA c < G2 (G2 = min(G, steps / 4): every range holds >= 4 key-tile steps).
struct AttnSched {
    int n_qt, n_kv, n_units, G;
    int R, rem, G2;
    long long U;                                   // key-tile steps of phase 2
    VCB_DEVICE void init(int n_heads, int n_tiles, int grid, int no_split = 0) {
        n_qt = n_tiles; n_kv = n_tiles; n_units = n_heads * n_qt; G = grid;
        R = n_units / G; rem = n_units - R * G;
        U = (long long)rem * n_kv;
        const long long g2 = U / 4;
        G2 = rem == 0 ? 0 : (int)(g2 < 1 ? 1 : (g2 < G ? g2 : G));
        if (no_split && rem > 0) G2 = rem;             // one whole unit per CTA c < rem: boundary(c) = c * n_kv
    }
    // start of CTA c's phase-2 range (c == G2: the end of the space)
    VCB_DEVICE void boundary(int c, int& unit, int& kv) const {
        const long long x = U * c / G2;
        const int ur = (int)(x / n_kv);
        unit = R * G + ur;
        kv = (int)(x - (long long)ur * n_kv);
    }
};

struct AttnSeg { int unit, kv0, kv1, n_parts; };

// enumerates CTA c's segments: phase 1 units, then the pieces of its phase-2 range.  n_parts (for a cut unit's finaliser) = the
// CTAs right after this one whose range starts inside the unit.
struct AttnSegIter {
    const AttnSched& s;
    int c, r, u, u_s, u_e, k_s, k_e;
    VCB_DEVICE AttnSegIter(const AttnSched& sched, int cta) : s(sched), c(cta), r(0) {
        if (c < s.G2) { s.boundary(c, u_s, k_s); s.boundary(c + 1, u_e, k_e); } else { u_s = 1; u_e = 0; k_s = k_e = 0; }
        u = u_s;
    }
    VCB_DEVICE bool next(AttnSeg& g) {
        if (r < s.R) { g.unit = r * s.G + c; g.kv0 = 0; g.kv1 = s.n_kv; g.n_parts = 0; ++r; return true; }
        while (u <= u_e && u < s.n_units) {
            const int cur = u++;
            const int kv0 = (cur == u_s) ? k_s : 0;
            const int kv1 = (cur == u_e) ? k_e : s.n_kv;
            if (kv0 >= kv1) continue;
            g.unit = cur; g.kv0 = kv0; g.kv1 = kv1; g.n_parts = 0;
            if (kv0 == 0 && kv1 < s.n_kv) {
                for (int pc = c + 1; pc < s.G2; ++pc) {
                    int pu, pk;
                    s.boundary(pc, pu, pk);
                    if (pu != cur) break;
                    ++g.n_parts;
                }
            }
            return true;
        }
        return false;
    }
};
// one entry of a CTA's segment list, computed once by one thread (keeps the 64-bit schedule arithmetic out of the role loops)
struct AttnSegEntry { int b, head, q0, kv0, kv1, seqlen, n_parts, unit; };
static_assert(sizeof(AttnSegEntry) == 32, "segment entry");

// CTA `cta`'s segment list -> shared memory; returns the count.  Out of line on purpose: its locals (iterator structs, 64-bit schedule
// arithmetic) get their own stack frame instead of forcing one on the kernel.
__device__ __noinline__ int attn4_build_segments(const AttnSched& sched, int cta, int heads, int seqlen, AttnSegEntry* segs) {
    AttnSegIter it(sched, cta);
    AttnSeg g;
    int n = 0;
    while (n < kAttn4MaxSegs && it.next(g)) {
        AttnSegEntry e;
        const int hi = g.unit / sched.n_qt;
        e.b = hi / heads;
        e.head = hi - e.b * heads;
        e.q0 = (g.unit - hi * sched.n_qt) * kAttnTile;
        e.kv0 = g.kv0; e.kv1 = g.kv1; e.unit = g.unit; e.n_parts = g.n_parts;
        e.seqlen = seqlen;
        segs[n++] = e;
    }
    return n;
}

VCB_DEVICE unsigned long long globaltimer_ns() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
    return t;
}
// mbarrier wait with a watchdog (segment-level waits only; the per-key-tile waits use the plain mbar_wait): a wait that never
// completes traps the kernel instead of hanging the GPU
VCB_DEVICE void mbar_wait_wd(uint64_t* bar, uint32_t parity) {
    if (mbar_try_wait(bar, parity)) return;
    uint32_t spins = 0;
    while (!mbar_try_wait(bar, parity)) {
        if (++spins > (1u << 26)) __trap();
    }
}

template <bool kFixed>
__global__ void __launch_bounds__(kAttnThreads, 1)
attn_fwd_wgmma_kernel(const __grid_constant__ CUtensorMap tmap_qkv, const AttnParams p, const AttnSkParams skp) {
    const uint32_t warp = warp_id_uniform();
    const uint32_t lane = lane_id();
    const bool persistent = skp.ws != nullptr;
    const int cta = blockIdx.x;
    pdl_launch_dependents();

    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint8_t* smem_q = smem;                                  // 32 KB: two [128 rows x 64 columns] blocks
    uint8_t* smem_kv = smem + kSlotBytes;
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + (1 + kAttnSlots) * kSlotBytes);
    uint64_t* q_full = bars;                       // [1]   one phase per segment
    uint64_t* q_empty = bars + 1;                  // [1]   all Q K^T of the segment have run: the Q tile may be overwritten
    uint64_t* kv_full = bars + 2;                  // [slots]
    uint64_t* kv_empty = kv_full + kAttnSlots;     // [slots]
    int* n_segs_smem = reinterpret_cast<int*>(kv_empty + kAttnSlots);
    AttnSegEntry* segs = reinterpret_cast<AttnSegEntry*>(smem + (1 + kAttnSlots) * kSlotBytes + 256);

    if (warp == 4 && lane == 0) {
        if (persistent) {
            AttnSched sched;
            sched.init(p.B * p.H, (p.L + kAttnTile - 1) / kAttnTile, gridDim.x, skp.no_split);
            *n_segs_smem = attn4_build_segments(sched, cta, p.H, p.L, segs);
        } else {
            const int b = blockIdx.z;
            const int seqlen = p.seqlens ? min(__ldg(p.seqlens + b), p.L) : p.L;
            segs[0] = AttnSegEntry{b, (int)blockIdx.y, (int)blockIdx.x * kAttnTile, 0, (seqlen + kAttnTile - 1) / kAttnTile, seqlen, 0, 0};
            *n_segs_smem = 1;
        }
    }
    if (warp == 0 && lane == 0) {
        tma_prefetch_desc(&tmap_qkv);
        mbar_init(q_full, 1);
        mbar_init(q_empty, 2);                      // one arrive per consumer warpgroup
        for (int s = 0; s < kAttnSlots; ++s) { mbar_init(&kv_full[s], 1); mbar_init(&kv_empty[s], 2); }
        fence_barrier_init();
    }
    __syncthreads();
    pdl_wait();                                     // everything above overlapped the previous kernel's tail

    const int n_segs = *n_segs_smem;
    const int n_kv_all = (p.L + kAttnTile - 1) / kAttnTile;
    if (skp.timeline != nullptr && warp == 4 && lane == 0) skp.timeline[(long long)cta * (kAttn4MaxSegs + 2)] = globaltimer_ns();

    if (warp < 4) {
        // ===================== TMA producer =====================
        setmaxnreg_dec<40>();
        if (warp == 0 && lane == 0) {
            int seq = 0;
            for (int segn = 0; segn < n_segs; ++segn) {
                const int b = segs[segn].b, head = segs[segn].head, q0 = segs[segn].q0, kv0 = segs[segn].kv0, kv1 = segs[segn].kv1;
                if (q0 >= segs[segn].seqlen) continue;                 // a tile of padding rows: the consumers write zeros
                if (segn > 0) mbar_wait_wd(q_empty, (uint32_t)(segn - 1) & 1u);
                mbar_expect_tx(q_full, kSlotBytes);
                tma_load_3d(&tmap_qkv, q_full, smem_q, p.q_col + head * 128, q0, b, kEvictFirst);
                tma_load_3d(&tmap_qkv, q_full, smem_q + kSlotBytes / 2, p.q_col + head * 128 + 64, q0, b, kEvictFirst);
                for (int e = 0; e < 2 * (kv1 - kv0); ++e, ++seq) {       // K V K V ...
                    const int slot = seq % kAttnSlots;
                    const uint32_t ph = (uint32_t)(seq / kAttnSlots) & 1u;
                    const int j = kv0 + (e >> 1);
                    const int col = ((e & 1) ? p.v_col : p.k_col) + head * 128;
                    mbar_wait(&kv_empty[slot], ph ^ 1);
                    mbar_expect_tx(&kv_full[slot], kSlotBytes);
                    uint8_t* dst = smem_kv + slot * kSlotBytes;
                    tma_load_3d(&tmap_qkv, &kv_full[slot], dst, col, j * kAttnTile, b, kEvictLast);
                    tma_load_3d(&tmap_qkv, &kv_full[slot], dst + kSlotBytes / 2, col + 64, j * kAttnTile, b, kEvictLast);
                }
            }
        }
    } else {
        // ===================== consumer warpgroups: 64 query rows each =====================
        setmaxnreg_inc<232>();
        const int ctid = (int)threadIdx.x - 128;
        const int wg = ctid >> 7;
        const uint32_t q = lane & 3;
        const int frag_row = wg * 64 + (int)(warp & 3) * 16 + (int)(lane >> 2);       // + 8 h
        const bool elected = (warp & 3) == 0 && lane == 0;
        const float sc = p.scale_log2;
        int seq = 0;
        for (int segn = 0; segn < n_segs; ++segn) {
            const int b = segs[segn].b, head = segs[segn].head, q0 = segs[segn].q0, kv0 = segs[segn].kv0, kv1 = segs[segn].kv1;
            const int seqlen = segs[segn].seqlen;
            if (q0 >= seqlen) {
                // the tile is padding (per-tile grid only): zero rows (pad_input)
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int row = q0 + frag_row + 8 * h;
                    if (row < p.L) {
                        uint4* dst = reinterpret_cast<uint4*>(attn_out_row(p, b, row) + p.out_col_offset + head * 128 + 8 * (int)q);
#pragma unroll
                        for (int c = 0; c < 4; ++c) dst[c * 4] = make_uint4(0, 0, 0, 0);
                    }
                }
                continue;
            }
            float o[64];
            [[maybe_unused]] float m_run[2] = {-INFINITY, -INFINITY};
            float l_run[2] = {0.f, 0.f};                     // this lane's share of the row sums (its own key columns)
            mbar_wait_wd(q_full, (uint32_t)segn & 1u);
            const uint64_t qd = make_smem_desc(smem_u32(smem_q + wg * 64 * 128), 16, 1024);
            for (int j = kv0; j < kv1; ++j, seq += 2) {
                const int k_slot = seq % kAttnSlots, v_slot = (seq + 1) % kAttnSlots;
                // ---- S = Q K_j^T ----
                float s[64];
                mbar_wait(&kv_full[k_slot], (uint32_t)(seq / kAttnSlots) & 1u);
                const uint64_t kd = make_smem_desc(smem_u32(smem_kv + k_slot * kSlotBytes), 16, 1024);
                wgmma_fence();
#pragma unroll
                for (int ks = 0; ks < 8; ++ks) {
                    // +32 B per 16-wide k step inside a 64-wide block, +16 KB for the second block (descriptor units of 16 B)
                    const uint64_t off = (uint64_t)(((ks >> 2) * (kSlotBytes / 2) + (ks & 3) * 32) >> 4);
                    wgmma_ss<128>(s, qd + off, kd + off, ks != 0);
                }
                wgmma_commit();
                wgmma_wait<0>();
                if (elected) {
                    mbar_arrive(&kv_empty[k_slot]);
                    if (j == kv1 - 1) mbar_arrive(q_empty);            // that was the segment's last Q K^T
                }
                // ---- softmax: s[4 jj + 2 h + e] is row frag_row + 8 h, key column 8 jj + 2 q + e ----
                const int kv_left = seqlen - j * kAttnTile;             // columns >= kv_left are padding
                if (kv_left < kAttnTile) {
#pragma unroll
                    for (int i = 0; i < 64; ++i)
                        if (8 * (i >> 2) + 2 * (int)q + (i & 1) >= kv_left) s[i] = -INFINITY;      // p = 0
                }
                float m_new[2] = {p.fixed_max, p.fixed_max};
                if constexpr (!kFixed) {
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        float m_tile = -INFINITY;
#pragma unroll
                        for (int jj = 0; jj < 16; ++jj) m_tile = fmaxf(m_tile, fmaxf(s[4 * jj + 2 * h], s[4 * jj + 2 * h + 1]));
                        m_tile = fmaxf(m_tile, __shfl_xor_sync(0xffffffffu, m_tile, 1));
                        m_tile = fmaxf(m_tile, __shfl_xor_sync(0xffffffffu, m_tile, 2));
                        m_new[h] = fmaxf(m_run[h], m_tile * sc);        // scaled log2 units; every key tile has a valid column
                        const float alpha = ex2_approx(m_run[h] - m_new[h]);
                        if (j > kv0) {
#pragma unroll
                            for (int jj = 0; jj < 16; ++jj) { o[4 * jj + 2 * h] *= alpha; o[4 * jj + 2 * h + 1] *= alpha; }
                        }
                        l_run[h] *= alpha;
                        m_run[h] = m_new[h];
                    }
                }
                uint32_t pa[8][4];                           // P as the A operand of P V: 8 k steps of 16 keys
#pragma unroll
                for (int jj = 0; jj < 16; ++jj) {
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        const float p0 = ex2_approx(fmaf(s[4 * jj + 2 * h], sc, -m_new[h]));
                        const float p1 = ex2_approx(fmaf(s[4 * jj + 2 * h + 1], sc, -m_new[h]));
                        l_run[h] += p0 + p1;
                        pa[jj >> 1][(jj & 1) * 2 + h] = pack_bf16x2(p0, p1);
                    }
                }
                // ---- O (+)= P V_j: V is MN-major (head dim contiguous): two [128 keys x 64] blocks, 16 keys = 2048 bytes ----
                mbar_wait(&kv_full[v_slot], (uint32_t)((seq + 1) / kAttnSlots) & 1u);
                // Padded keys of a right-padded sample's last tile: their P entries are exactly 0, but the tensor core's 0 * NaN and
                // 0 * Inf are NaN, and the padded V rows hold whatever the caller left there (they lie inside L, so the TMA unit loads
                // them; rows >= L arrive zero-filled).  Zero them first: whole 128-byte rows of both 64-column blocks, independent of
                // the swizzle.  Both warpgroups read the slot, so both take part and meet at a barrier after the proxy fence.
                if (kv_left < kAttnTile && seqlen < p.L) {
                    const int n_pad = min(kAttnTile, p.L - j * kAttnTile) - kv_left;           // uint4 per row: 8
                    uint4* vs = reinterpret_cast<uint4*>(smem_kv + v_slot * kSlotBytes);
                    for (int i = ctid; i < 2 * n_pad * 8; i += kAttnConsumers) {
                        const int half = i / (n_pad * 8), r = i - half * (n_pad * 8);
                        vs[half * (kSlotBytes / 32) + (kv_left + (r >> 3)) * 8 + (r & 7)] = make_uint4(0, 0, 0, 0);
                    }
                    fence_proxy_async_smem();                       // generic-proxy stores -> visible to the wgmma (async proxy)
                    named_bar_sync(1, kAttnConsumers);
                }
                const uint64_t vd = make_smem_desc(smem_u32(smem_kv + v_slot * kSlotBytes), kSlotBytes / 2, 1024);
                wgmma_fence();
#pragma unroll
                for (int ks = 0; ks < 8; ++ks) wgmma_rs<128, true>(o, pa[ks], vd + (uint64_t)(ks * (2048 >> 4)), (j > kv0 || ks != 0) ? 1u : 0u);
                wgmma_commit();
                wgmma_wait<0>();
                if (elected) mbar_arrive(&kv_empty[v_slot]);
            }

            // ---------------- segment epilogue ----------------
#pragma unroll
            for (int h = 0; h < 2; ++h) l_run[h] = quad_sum(l_run[h]);
            const bool contributor = kv0 > 0;                 // not the piece holding key tile 0: dump partials
            if (contributor) {
                // un-normalised O (fp32, register-major: consecutive threads write consecutive words), row sums and reference exponents
                float* my_slot = skp.ws + (long long)cta * kAttn4SlotFloats;
#pragma unroll
                for (int i = 0; i < 64; ++i) my_slot[i * kAttnConsumers + ctid] = o[i];
                if (q == 0) {
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        my_slot[128 * 128 + frag_row + 8 * h] = l_run[h];
                        if constexpr (!kFixed) my_slot[128 * 128 + 128 + frag_row + 8 * h] = m_run[h];
                    }
                }
                // every consumer thread of the CTA has written (and fenced) its part of the slot -> publish
                __threadfence();
                named_bar_sync(1, kAttnConsumers);
                if (ctid == 0) st_release_gpu(skp.flags + cta, skp.epoch);
            } else {
                // fold the other pieces of this unit (the CTAs right after this one whose range starts inside it), normalise, store
                const int n_parts = kv1 < n_kv_all ? segs[segn].n_parts : 0;
                if (n_parts > 0) {
                    if (lane == 0) {
                        for (int pc = cta + 1; pc <= cta + n_parts; ++pc) {
                            uint32_t spins = 0;
                            while (ld_acquire_gpu(skp.flags + pc) != skp.epoch) {
                                if (++spins > (1u << 28)) __trap();
                            }
                        }
                    }
                    __syncwarp();
                    float a_own[2] = {1.f, 1.f};
                    [[maybe_unused]] float m_fin[2] = {m_run[0], m_run[1]};
                    if constexpr (!kFixed) {
#pragma unroll
                        for (int h = 0; h < 2; ++h) {
                            for (int i = 1; i <= n_parts; ++i)
                                m_fin[h] = fmaxf(m_fin[h], __ldcg(skp.ws + (long long)(cta + i) * kAttn4SlotFloats + 128 * 128 + 128 + frag_row + 8 * h));
                            a_own[h] = ex2_approx(m_run[h] - m_fin[h]);
                            l_run[h] *= a_own[h];
                        }
#pragma unroll
                        for (int i = 0; i < 64; ++i) o[i] *= a_own[(i >> 1) & 1];
                    }
                    for (int pi = 1; pi <= n_parts; ++pi) {
                        const float* pslot = skp.ws + (long long)(cta + pi) * kAttn4SlotFloats;
                        float ap[2] = {1.f, 1.f};
#pragma unroll
                        for (int h = 0; h < 2; ++h) {
                            if constexpr (!kFixed) ap[h] = ex2_approx(__ldcg(pslot + 128 * 128 + 128 + frag_row + 8 * h) - m_fin[h]);
                            l_run[h] = fmaf(__ldcg(pslot + 128 * 128 + frag_row + 8 * h), ap[h], l_run[h]);
                        }
#pragma unroll
                        for (int i = 0; i < 64; ++i) o[i] = fmaf(__ldcg(pslot + i * kAttnConsumers + ctid), ap[(i >> 1) & 1], o[i]);
                    }
                }
#pragma unroll
                for (int c = 0; c < 4; ++c) {
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        float v[8];
                        frag_row8(o, c, h, q, v);
                        const int row = q0 + frag_row + 8 * h;
                        if (row < p.L) {
                            // padded query rows: +0 (pad_input) as a select -- their o may be NaN when Q holds NaN there
                            const bool valid = row < seqlen;
                            const float inv_l = 1.0f / l_run[h];
#pragma unroll
                            for (int i = 0; i < 8; ++i) v[i] = valid ? v[i] * inv_l : 0.f;
                            store_bf16x8(attn_out_row(p, b, row) + p.out_col_offset + head * 128 + c * 32 + 8 * (int)q, v);
                        }
                    }
                }
            }
            if (skp.timeline != nullptr && ctid == 0) skp.timeline[(long long)cta * (kAttn4MaxSegs + 2) + 1 + segn] = globaltimer_ns();
        }
    }
}

}  // namespace vcb
