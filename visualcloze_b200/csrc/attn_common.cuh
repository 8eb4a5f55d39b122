// attn_common.cuh -- parameters and constants of the joint-attention kernel (attn_sm90.cuh: one CTA per query tile, or the
// persistent schedule).
//
// Contract (models/math.py:63-99: attention -> _upad_input -> flash_attn_varlen_func -> pad_input): non-causal
// softmax(Q K^T / sqrt(128)) V over right-padded samples, head_dim 128, bf16 in / fp32 accumulate / bf16 out.  Padding is handled
// with per-sample `seqlens` instead of the reference's gather/scatter unpad: keys >= seqlen are masked to -inf, query rows >=
// seqlen produce zeros (pad_input semantics).  RoPE and QK-RMSNorm are already applied by the QKV GEMM epilogue.
#pragma once
#include "vcb_common.cuh"

namespace vcb {

struct AttnParams {
    int B, L, H;                 // samples, padded tokens per sample, heads
    const int* seqlens;          // [B] valid tokens per sample (<= L); null = all L
    __nv_bfloat16* out;          // [B*L, ldo], head h at columns out_col_offset + h*128
    long long ldo;
    int out_col_offset;
    int q_col, k_col, v_col;     // column of head 0 of q / k / v inside the qkv matrix
    float scale_log2;            // head_dim^-0.5 * log2(e)
    float fixed_max;             // > 0: upper bound of |score * scale_log2| guaranteed by the caller (kFixed)
    // Sequence-parallel output routing (B == 1; sp_world <= 1 = off): query row r belongs to rank
    // r / sp_rows and is stored over NVLink into that rank's peer-mapped buffer sp_out[rank] at row r % sp_rows.
    int sp_world, sp_rows;
    __nv_bfloat16* sp_out[8];
};

// first element of output row `row` of sample b (columns are added by the caller)
VCB_DEVICE __nv_bfloat16* attn_out_row(const AttnParams& p, int b, int row) {
    if (p.sp_world > 1) {
        const int owner = min(row / p.sp_rows, p.sp_world - 1);
        return p.sp_out[owner] + (long long)(row - owner * p.sp_rows) * p.ldo;
    }
    return p.out + ((long long)b * p.L + row) * p.ldo;
}

constexpr int kAttnTile = 128;           // query rows per CTA == kv rows per tile == head_dim
constexpr int kSlotBytes = 128 * 128 * 2;
constexpr float kRescaleThreshold = 8.0f;   // log2 units: only rescale O when the row max grows by > 2^8

}  // namespace vcb
