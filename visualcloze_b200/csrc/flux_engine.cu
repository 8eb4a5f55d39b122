// flux_engine.cu -- Flux.forward (models/model.py:85-124) as a fixed sequence of libvcb200 kernel launches.
//
// Data layout in HBM (all bf16 unless noted), B samples, L = Lt + Li tokens per sample, txt rows first:
//   x    [B, L, H]         residual stream of both streams (the reference keeps img/txt apart and cats them at
//                          model.py:116; here the double blocks address their stream through row offsets)
//   xm   [B, L, H]         AdaLN-modulated LayerNorm output (GEMM A operand)
//   qkv  [B, L, 3H]        q | k | v after bias, QK-RMSNorm and RoPE (GEMM epilogue) -> attention operand
//   cat  [B, L, H + mlp]   columns [0,H): attention output; [H,H+mlp): GELU(mlp-up)  == linear2 input (layers.py:244)
//   rope [64][B*L] float2 (pair-major), txt0 [B, Lt, H] (txt_in output), modulation tables for all evaluations.
// Step-invariant work is hoisted into vcb_flux_prepare (SURVEY.md 7.5).
#include <algorithm>
#include <cmath>
#include <vector>

#include "../../include/vcb200.h"
#include "fbcache.cuh"
#include "host_util.cuh"

using namespace vcb;

struct vcb_flux {
    vcb_flux_config cfg;
    vcb_flux_weights w;
    std::vector<vcb_double_w> dbl;
    std::vector<vcb_single_w> sgl;
    // prepared state
    bool prepared = false;
    int B = 0, Li = 0, Lt = 0, L = 0, E = 0;
    bool use_score_bounds = true;
    int fp8 = 0;                      // vcb_flux_set_fp8 level: 1 = LayerNorm-fed projections on e4m3 operands, 2 = every block Linear
    uint8_t* cat8 = nullptr;          // [B, L, H + mlp] e4m3 copy of `cat` (level 2)
    float* cat_scale = nullptr;       // [B * L] fp32 per-row scale of the cat8 columns last quantised (level 2)
    uint8_t* xm8 = nullptr;           // [B, L, H] e4m3 LayerNorm output (fp8 mode)
    float* row_scale = nullptr;       // [B * L] fp32 per-row activation scale (fp8 mode)
    float* row_stats = nullptr;       // [B * L][H / 64] float2: LayerNorm statistics left behind by the GATE_RES epilogues
    bool stats_valid = false;         // row_stats describes the current x (false right after img_in / the txt copy)     // false: every block runs the exact online-max softmax (vcb_flux_use_score_bounds)
    const int32_t* seqlens = nullptr;
    float2* rope = nullptr;
    uint16_t *txt0 = nullptr, *temb_t = nullptr, *temb_g = nullptr, *h1 = nullptr, *e_time = nullptr, *e_guid = nullptr,
             *e_vec = nullptr, *vec = nullptr, *svec = nullptr, *mod_final = nullptr, *x = nullptr, *xm = nullptr,
             *qkv = nullptr, *cat = nullptr;
    std::vector<uint16_t*> mod_dbl;   // [depth * 2] (img, txt), each [E*B, 6H]
    std::vector<uint16_t*> mod_sgl;   // [depth_single], each [E*B, 3H]
    // sequence-parallel mode (vcb_flux_sp_attach): W ranks share one sample; qkv / cat live in peer-mapped buffers
    int sp_world = 1, sp_rank = 0, sp_epoch = 0, sp_timeout_ms = 2000;
    void* sp_qkv[VCB_SP_MAX] = {};
    void* sp_cat[VCB_SP_MAX] = {};
    int32_t* sp_flags[VCB_SP_MAX] = {};
    int32_t* sp_err = nullptr;
    // unmerged LoRA: the largest rank of the Linears that carry one (0 = every Linear merged) and the down-projection buffer
    // T [max(B * L, E * B), lora_rmax] bf16, written by each LoRA Linear's down-projection and read by its k-tail right after
    int lora_rmax = 0;
    uint16_t* lora_t = nullptr;
    // first-block cache (vcb_flux_set_first_block_cache_ex; threshold 0 = off).  fbc_buf[fbc_ref] holds r_ref, the block-0
    // residual of the last computed evaluation; the other one takes the x0 copy, which the decision turns into r_k in place -- an
    // evaluation computed for every sample then swaps the two and parks x1 in the freed one until the residual R is stored.  When
    // only some samples compute (per-sample mode), their rows of r_k are copied into r_ref instead and x1 overwrites r_k.
    float fbc_threshold = 0.f;
    bool fbc_per_sample = false;      // one decision per sample instead of one per batch
    uint16_t* fbc_buf[2] = {};        // [B * Li, H] bf16 each
    int fbc_ref = 0;
    float* fbc_R = nullptr;           // [B * Li, H] fp32: x_final - x1 of the last computed evaluation (per sample)
    float2* fbc_part = nullptr;       // [kFbcMaxBlocks] partial sums of the decision
    float* fbc_res = nullptr;         // [4 * groups + 1] per group num, den, diff, skip; then the number of skipping groups (device)
    float* fbc_host = nullptr;        // pinned copy of fbc_res read by the host
    int fbc_host_cap = 0;             // floats fbc_host holds
    int32_t fbc_computed = 0, fbc_skipped = 0;
    float fbc_last_diff = NAN;
    std::vector<int32_t> fbc_s_computed, fbc_s_skipped;    // [B] per-sample counters (per-sample mode)
    std::vector<float> fbc_s_diff;                         // [B] latest per-sample diff
    std::vector<char> fbc_s_skip;                          // [B] this evaluation's per-sample decision
    ~vcb_flux() { if (fbc_host) cudaFreeHost(fbc_host); }
};

namespace {

struct Carver {
    uint8_t* base;
    int64_t off = 0;
    template <class T>
    T* take(int64_t count) {
        T* p = base ? reinterpret_cast<T*>(base + off) : nullptr;
        off += ((count * (int64_t)sizeof(T) + 255) / 256) * 256;
        return p;
    }
};

// carve the workspace; with base == nullptr only the size is computed
int64_t carve(vcb_flux* f, uint8_t* base, int B, int Li, int Lt, int E) {
    const vcb_flux_config& c = f->cfg;
    const int64_t H = c.hidden, L = Li + Lt, EB = (int64_t)E * B;
    Carver cv{base};
    float2* rope = cv.take<float2>((int64_t)B * L * 64);
    uint16_t* txt0 = cv.take<uint16_t>((int64_t)B * Lt * H);
    uint16_t* temb_t = cv.take<uint16_t>(EB * 256);
    uint16_t* temb_g = cv.take<uint16_t>((int64_t)B * 256);
    uint16_t* h1 = cv.take<uint16_t>(EB * H);
    uint16_t* e_time = cv.take<uint16_t>(EB * H);
    uint16_t* e_guid = cv.take<uint16_t>((int64_t)B * H);
    uint16_t* e_vec = cv.take<uint16_t>((int64_t)B * H);
    uint16_t* vec = cv.take<uint16_t>(EB * H);
    uint16_t* svec = cv.take<uint16_t>(EB * H);
    std::vector<uint16_t*> md(c.depth * 2), ms(c.depth_single);
    for (auto& p : md) p = cv.take<uint16_t>(EB * 6 * H);
    for (auto& p : ms) p = cv.take<uint16_t>(EB * 3 * H);
    uint16_t* mod_final = cv.take<uint16_t>(EB * 2 * H);
    uint16_t* x = cv.take<uint16_t>((int64_t)B * L * H);
    uint16_t* xm = cv.take<uint16_t>((int64_t)B * L * H);
    uint8_t* xm8 = cv.take<uint8_t>((int64_t)B * L * H);
    float* row_scale = cv.take<float>((int64_t)B * L);
    uint8_t* cat8 = cv.take<uint8_t>(f->fp8 >= 2 ? (int64_t)B * L * (H + f->cfg.mlp_hidden) : 0);
    float* cat_scale = cv.take<float>(f->fp8 >= 2 ? (int64_t)B * L : 0);
    float* row_stats = cv.take<float>((int64_t)B * L * (H / 64) * 2);
    uint16_t* lora_t = cv.take<uint16_t>(f->lora_rmax ? std::max<int64_t>((int64_t)B * L, EB) * f->lora_rmax : 0);
    const int64_t fbc_n = f->fbc_threshold > 0.f ? (int64_t)B * Li * H : 0;
    uint16_t* fbc_b0 = cv.take<uint16_t>(fbc_n);
    uint16_t* fbc_b1 = cv.take<uint16_t>(fbc_n);
    float* fbc_R = cv.take<float>(fbc_n);
    float2* fbc_part = cv.take<float2>(fbc_n ? kFbcMaxBlocks : 0);
    float* fbc_res = cv.take<float>(fbc_n ? 4 * (f->fbc_per_sample ? B : 1) + 1 : 0);
    // sequence-parallel: qkv [W*L, 3H/W] and cat [L, H+mlp] are the caller's peer-mapped allocations (same sizes)
    const bool sp = f->sp_world > 1;
    uint16_t* qkv = sp ? static_cast<uint16_t*>(f->sp_qkv[f->sp_rank]) : cv.take<uint16_t>((int64_t)B * L * 3 * H);
    uint16_t* cat = sp ? static_cast<uint16_t*>(f->sp_cat[f->sp_rank]) : cv.take<uint16_t>((int64_t)B * L * (H + c.mlp_hidden));
    if (base) {
        f->rope = rope; f->txt0 = txt0; f->temb_t = temb_t; f->temb_g = temb_g; f->h1 = h1; f->e_time = e_time;
        f->e_guid = e_guid; f->e_vec = e_vec; f->vec = vec; f->svec = svec; f->mod_dbl = md; f->mod_sgl = ms;
        f->mod_final = mod_final; f->x = x; f->xm = xm; f->qkv = qkv; f->cat = cat; f->xm8 = xm8; f->row_scale = row_scale; f->row_stats = row_stats;
        f->cat8 = cat8; f->cat_scale = cat_scale; f->lora_t = lora_t;
        f->fbc_buf[0] = fbc_b0; f->fbc_buf[1] = fbc_b1; f->fbc_R = fbc_R; f->fbc_part = fbc_part; f->fbc_res = fbc_res;
    }
    return cv.off;
}

bool has_lora(const vcb_linear_w& w) { return w.rank > 0 && w.lora_scale != 0.f; }

// One Linear, or two (the img and txt streams of a double block) in one grouped launch.  An unmerged LoRA Linear first runs its
// down-projection T = bf16(s * A lora_a^T) into the T buffer, at the rows the main GEMM writes (the joint-row mapping of its A
// operand; both streams' down-projections share one grouped launch), then the main GEMM reads T back through its LoRA k-tail.
int gemm_linear(const vcb_flux* f, vcb_gemm_args* g, const vcb_linear_w* const* w, int n, void* stream) {
    if (has_lora(*w[0]) || (n == 2 && has_lora(*w[1]))) {
        vcb_gemm_args d[2];
        for (int s = 0; s < n; ++s) {
            const int r = w[s]->rank;
            d[s] = vcb_gemm_args{};
            d[s].M = g[s].M; d[s].N = r; d[s].K = g[s].K;
            d[s].A = g[s].A; d[s].lda = g[s].lda; d[s].a_batch_stride = g[s].a_batch_stride;
            d[s].W = w[s]->lora_a; d[s].ldw = g[s].K;
            d[s].out = f->lora_t; d[s].ldo = r;
            d[s].rows_per_batch = g[s].rows_per_batch; d[s].out_batch_rows = g[s].out_batch_rows; d[s].out_row_offset = g[s].out_row_offset;
            d[s].epilogue = VCB_EPI_BIAS;
            d[s].alpha = w[s]->lora_scale;
            g[s].lora_t = f->lora_t + (int64_t)g[s].out_row_offset * r; g[s].ld_lora_t = r;
            g[s].lora_t_batch_stride = (int64_t)g[s].out_batch_rows * r;
            g[s].lora_b = w[s]->lora_b; g[s].lora_rank = r;
        }
        if (int rc = n == 2 ? vcb_gemm_bf16_grouped(&d[0], &d[1], stream) : vcb_gemm_bf16(&d[0], stream)) return rc;
    }
    return n == 2 ? vcb_gemm_bf16_grouped(&g[0], &g[1], stream) : vcb_gemm_bf16(&g[0], stream);
}

int gemm_linear(const vcb_flux* f, vcb_gemm_args& g, const vcb_linear_w& w, void* stream) {
    const vcb_linear_w* wp = &w;
    return gemm_linear(f, &g, &wp, 1, stream);
}

// plain [M,K] x [N,K]^T GEMM through the public entry point
int linear(const vcb_flux* f, const void* A, int64_t lda, int M, int K, const vcb_linear_w& w, int N, void* out, int64_t ldo, int epi,
           void* stream) {
    vcb_gemm_args g{};
    g.M = M; g.N = N; g.K = K;
    g.A = A; g.lda = lda;
    g.W = w.w; g.ldw = K; g.bias = w.b;
    g.out = out; g.ldo = ldo;
    g.rows_per_batch = M; g.out_batch_rows = M;
    g.epilogue = epi;
    return gemm_linear(f, g, w, stream);
}

}  // namespace

extern "C" int vcb_flux_create(const vcb_flux_config* cfg, const vcb_flux_weights* w, vcb_flux** out) {
    if (!cfg || !w || !out) return set_error("flux_create: null argument");
    if (cfg->hidden != cfg->heads * 128) return set_error("flux_create: head_dim must be 128 (hidden = heads * 128)");
    if (cfg->hidden % 256) return set_error("flux_create: hidden must be a multiple of 256");
    if (cfg->axes_dim[0] + cfg->axes_dim[1] + cfg->axes_dim[2] != 128) return set_error("flux_create: axes_dim must sum to 128");
    if (cfg->in_channels % 8 || cfg->out_channels % 8 || cfg->vec_in_dim % 8 || cfg->context_in_dim % 8 || cfg->mlp_hidden % 128)
        return set_error("flux_create: channel counts must be multiples of 8 (mlp_hidden of 128)");
    if (cfg->depth < 0 || cfg->depth_single < 0 || (cfg->depth && !w->dbl) || (cfg->depth_single && !w->sgl))
        return set_error("flux_create: missing block weights");
    // unmerged LoRA Linears: validate, and size the down-projection buffer by the largest rank
    int rmax = 0;
    std::vector<const vcb_linear_w*> all = {&w->img_in, &w->txt_in, &w->time_in0, &w->time_in1, &w->vector_in0, &w->vector_in1,
                                            &w->final_mod, &w->final_linear};
    if (cfg->guidance_embed) { all.push_back(&w->guidance_in0); all.push_back(&w->guidance_in1); }
    for (int i = 0; i < cfg->depth; ++i)
        for (const vcb_stream_w* s : {&w->dbl[i].img, &w->dbl[i].txt})
            for (const vcb_linear_w* l : {&s->mod, &s->qkv, &s->proj, &s->mlp0, &s->mlp2}) all.push_back(l);
    for (int i = 0; i < cfg->depth_single; ++i)
        for (const vcb_linear_w* l : {&w->sgl[i].mod, &w->sgl[i].linear1, &w->sgl[i].linear2}) all.push_back(l);
    for (const vcb_linear_w* l : all) {
        if (l->rank < 0 || l->rank % 8) return set_error("flux_create: LoRA rank %d must be a non-negative multiple of 8", l->rank);
        if (!has_lora(*l)) continue;
        if (!l->lora_a || !l->lora_b) return set_error("flux_create: an unmerged LoRA Linear (rank > 0) needs lora_a and lora_b");
        rmax = std::max(rmax, (int)l->rank);
    }
    vcb_flux* f = new vcb_flux();
    f->cfg = *cfg;
    f->lora_rmax = rmax;
    f->w = *w;
    f->dbl.assign(w->dbl, w->dbl + cfg->depth);
    f->sgl.assign(w->sgl, w->sgl + cfg->depth_single);
    f->w.dbl = f->dbl.data();
    f->w.sgl = f->sgl.data();
    *out = f;
    return 0;
}

extern "C" void vcb_flux_destroy(vcb_flux* f) { delete f; }

extern "C" int vcb_flux_set_fp8(vcb_flux* f, int32_t level) {
    if (!f) return set_error("flux_set_fp8: null engine");
    if (level < VCB_FP8_OFF || level > VCB_FP8_ALL_LINEARS) return set_error("flux_set_fp8: level must be 0 (off), 1 (LayerNorm-fed Linears) or 2 (all block Linears)");
    if (level) {
        if (f->sp_world > 1) return set_error("flux_set_fp8: the sequence-parallel mode runs bf16 projections");
        if (f->lora_rmax) return set_error("flux_set_fp8: unmerged LoRA Linears run on bf16 operands (merge the LoRA weights for fp8)");
        auto has8 = [](const vcb_linear_w& w) { return w.w8 && w.w8_scale; };
        for (const auto& d : f->dbl)
            for (const vcb_stream_w* s : {&d.img, &d.txt}) {
                if (!has8(s->qkv) || !has8(s->mlp0))
                    return set_error("flux_set_fp8: double-block qkv / mlp.0 weights carry no e4m3 copy (w8, w8_scale)");
                if (level >= 2 && (!has8(s->proj) || !has8(s->mlp2)))
                    return set_error("flux_set_fp8: level 2 needs e4m3 copies of the double-block attn.proj / mlp.2 weights too");
            }
        for (const auto& g : f->sgl) {
            if (!has8(g.linear1)) return set_error("flux_set_fp8: linear1 weights carry no e4m3 copy (w8, w8_scale)");
            if (level >= 2 && !has8(g.linear2)) return set_error("flux_set_fp8: level 2 needs an e4m3 copy of the linear2 weights too");
        }
        if (level >= 2 && (f->cfg.hidden + f->cfg.mlp_hidden > 15360 || f->cfg.hidden % 16 || f->cfg.mlp_hidden % 16))
            return set_error("flux_set_fp8: level 2 quantises rows of up to 15360 columns (hidden + mlp_hidden), both multiples of 16");
    }
    if (f->fp8 != level) f->prepared = false;       // the workspace layout depends on the level
    f->fp8 = level;
    return 0;
}

extern "C" int vcb_flux_set_first_block_cache_ex(vcb_flux* f, float threshold, int32_t per_sample) {
    if (!f) return set_error("flux_set_first_block_cache: null engine");
    if (!std::isfinite(threshold) || threshold < 0.f) return set_error("flux_set_first_block_cache: threshold must be a finite number >= 0 (0 = off)");
    if (per_sample != 0 && per_sample != 1) return set_error("flux_set_first_block_cache: per_sample must be 0 (one decision per batch) or 1");
    if (threshold > 0.f) {
        if (f->sp_world > 1) return set_error("flux_set_first_block_cache: the skip decision would have to agree across the sequence-parallel ranks");
        if (f->cfg.depth < 1) return set_error("flux_set_first_block_cache: the cache decides after the first double block (depth >= 1)");
    }
    // the workspace layout depends on whether the cache is on and, while on, on the mode
    if ((threshold > 0.f) != (f->fbc_threshold > 0.f) || (threshold > 0.f && (per_sample != 0) != f->fbc_per_sample)) f->prepared = false;
    f->fbc_threshold = threshold;
    f->fbc_per_sample = per_sample != 0;
    return 0;
}

extern "C" int vcb_flux_set_first_block_cache(vcb_flux* f, float threshold) { return vcb_flux_set_first_block_cache_ex(f, threshold, 0); }

extern "C" int vcb_flux_cache_stats(const vcb_flux* f, int32_t* computed, int32_t* skipped, float* last_diff) {
    if (!f || !computed || !skipped || !last_diff) return set_error("flux_cache_stats: null argument");
    *computed = f->fbc_computed; *skipped = f->fbc_skipped; *last_diff = f->fbc_last_diff;
    return 0;
}

extern "C" int vcb_flux_cache_stats_per_sample(const vcb_flux* f, int32_t B, int32_t* computed, int32_t* skipped, float* last_diff) {
    if (!f || !computed || !skipped || !last_diff) return set_error("flux_cache_stats_per_sample: null argument");
    if (!f->prepared) return set_error("flux_cache_stats_per_sample: call vcb_flux_prepare first");
    if (B != f->B) return set_error("flux_cache_stats_per_sample: B (%d) must be the prepared batch (%d)", B, f->B);
    const bool own = f->fbc_per_sample && f->fbc_threshold > 0.f;
    for (int b = 0; b < B; ++b) {          // per-batch mode: every sample shares the batch's decisions
        computed[b] = own ? f->fbc_s_computed[b] : f->fbc_computed;
        skipped[b] = own ? f->fbc_s_skipped[b] : f->fbc_skipped;
        last_diff[b] = own ? f->fbc_s_diff[b] : f->fbc_last_diff;
    }
    return 0;
}

extern "C" int vcb_flux_use_score_bounds(vcb_flux* f, int32_t enable) {
    if (!f) return set_error("flux_use_score_bounds: null engine");
    f->use_score_bounds = enable != 0;
    return 0;
}

extern "C" int64_t vcb_flux_workspace_bytes(const vcb_flux* f, int32_t B, int32_t Li, int32_t Lt, int32_t n_evals) {
    if (!f || B <= 0 || Li <= 0 || Lt < 0 || n_evals <= 0) return -1;
    return carve(const_cast<vcb_flux*>(f), nullptr, B, Li, Lt, n_evals);
}

extern "C" int vcb_flux_sp_shared_bytes(const vcb_flux* f, int32_t Li_local, int32_t Lt_local, int64_t* qkv_bytes, int64_t* cat_bytes) {
    if (!f || Li_local <= 0 || Lt_local < 0 || !qkv_bytes || !cat_bytes) return set_error("flux_sp_shared_bytes: bad arguments");
    const int64_t L = (int64_t)Li_local + Lt_local, H = f->cfg.hidden;
    *qkv_bytes = L * 3 * H * 2;                       // [W * L, 3H / W] bf16
    *cat_bytes = L * (H + f->cfg.mlp_hidden) * 2;
    return 0;
}

extern "C" int vcb_flux_sp_attach(vcb_flux* f, int32_t world, int32_t rank, void* const* qkv, void* const* cat,
                                  int32_t* const* flags, int32_t* err, int32_t timeout_ms) {
    if (!f) return set_error("flux_sp_attach: null engine");
    f->prepared = false;
    if (world <= 1) {
        f->sp_world = 1; f->sp_rank = 0;
        return 0;
    }
    if (world > VCB_SP_MAX || rank < 0 || rank >= world || !qkv || !cat || !flags || !err)
        return set_error("flux_sp_attach: bad arguments (world <= %d)", VCB_SP_MAX);
    if (f->cfg.heads % world) return set_error("flux_sp_attach: heads (%d) must be a multiple of world (%d)", f->cfg.heads, world);
    if (f->fp8) return set_error("flux_sp_attach: the sequence-parallel mode runs bf16 projections (switch vcb_flux_set_fp8 off first)");
    if (f->lora_rmax) return set_error("flux_sp_attach: the sequence-parallel mode takes merged LoRA weights only");
    if (f->fbc_threshold > 0.f) return set_error("flux_sp_attach: the first-block cache decides per batch on one device (switch it off first)");
    for (int r = 0; r < world; ++r) {
        if (!qkv[r] || !cat[r] || !flags[r]) return set_error("flux_sp_attach: null buffer for rank %d", r);
        f->sp_qkv[r] = qkv[r]; f->sp_cat[r] = cat[r]; f->sp_flags[r] = flags[r];
    }
    f->sp_world = world; f->sp_rank = rank; f->sp_err = err; f->sp_epoch = 0;
    f->sp_timeout_ms = timeout_ms > 0 ? timeout_ms : 2000;
    return 0;
}

extern "C" int vcb_flux_prepare(vcb_flux* f, void* workspace, int64_t workspace_bytes, int32_t B, int32_t Li, int32_t Lt,
                                int32_t n_evals, const void* txt, const void* y, const float* ids, const float* t_scaled,
                                const float* g_scaled, const float* freqs, const int32_t* seqlens, void* stream) {
    if (!f || !workspace || !txt || !y || !ids || !t_scaled || !freqs) return set_error("flux_prepare: null argument");
    if (B <= 0 || Li <= 0 || Lt <= 0 || n_evals <= 0) return set_error("flux_prepare: bad sizes");
    const vcb_flux_config& c = f->cfg;
    if (c.guidance_embed && !g_scaled) return set_error("Didn't get guidance strength for guidance distilled model.");
    if (f->sp_world > 1 && (B != 1 || seqlens)) return set_error("flux_prepare: sequence-parallel mode takes one unpadded sample (B == 1, seqlens NULL)");
    if ((reinterpret_cast<uintptr_t>(workspace) & 255) != 0) return set_error("flux_prepare: workspace must be 256-byte aligned");
    const int64_t need = carve(f, nullptr, B, Li, Lt, n_evals);
    if (workspace_bytes < need) return set_error("flux_prepare: workspace too small (%lld < %lld)", (long long)workspace_bytes, (long long)need);
    carve(f, static_cast<uint8_t*>(workspace), B, Li, Lt, n_evals);
    f->B = B; f->Li = Li; f->Lt = Lt; f->L = Li + Lt; f->E = n_evals; f->seqlens = seqlens;
    f->prepared = false;
    f->fbc_ref = 0; f->fbc_computed = 0; f->fbc_skipped = 0; f->fbc_last_diff = NAN;
    f->fbc_s_computed.assign(B, 0); f->fbc_s_skipped.assign(B, 0); f->fbc_s_diff.assign(B, NAN); f->fbc_s_skip.assign(B, 0);
    if (f->fbc_threshold > 0.f) {
        const int groups = f->fbc_per_sample ? B : 1;
        if (groups > kFbcMaxBlocks) return set_error("flux_prepare: the per-sample first-block cache takes at most %d samples", kFbcMaxBlocks);
        if (f->fbc_host_cap < 4 * groups + 1) {         // where vcb_flux_forward reads the cache's decision
            if (f->fbc_host) cudaFreeHost(f->fbc_host);
            f->fbc_host = nullptr; f->fbc_host_cap = 0;
            cudaError_t e = cudaMallocHost(reinterpret_cast<void**>(&f->fbc_host), (4 * groups + 1) * sizeof(float));
            if (e != cudaSuccess) { f->fbc_host = nullptr; return set_error("flux_prepare: pinned memory: %s", cudaGetErrorString(e)); }
            f->fbc_host_cap = 4 * groups + 1;
        }
    }
    const int H = c.hidden, EB = n_evals * B;
    int rc;
    // RoPE table (constant across steps; the reference recomputes it per call, model.py:110-111)
    if ((rc = vcb_rope_table(ids, f->rope, B * f->L, c.axes_dim[0], c.axes_dim[1], c.axes_dim[2], c.theta, stream))) return rc;
    // txt_in (constant across steps, model.py:108)
    if ((rc = linear(f, txt, c.context_in_dim, B * Lt, c.context_in_dim, f->w.txt_in, H, f->txt0, H, VCB_EPI_BIAS, stream))) return rc;
    // vec for every evaluation (model.py:102-107)
    if ((rc = vcb_timestep_embedding(t_scaled, freqs, f->temb_t, EB, stream))) return rc;
    if ((rc = linear(f, f->temb_t, 256, EB, 256, f->w.time_in0, H, f->h1, H, VCB_EPI_BIAS, stream))) return rc;
    if ((rc = vcb_silu(f->h1, f->h1, (int64_t)EB * H, stream))) return rc;
    if ((rc = linear(f, f->h1, H, EB, H, f->w.time_in1, H, f->e_time, H, VCB_EPI_BIAS, stream))) return rc;
    if (c.guidance_embed) {
        if ((rc = vcb_timestep_embedding(g_scaled, freqs, f->temb_g, B, stream))) return rc;
        if ((rc = linear(f, f->temb_g, 256, B, 256, f->w.guidance_in0, H, f->h1, H, VCB_EPI_BIAS, stream))) return rc;
        if ((rc = vcb_silu(f->h1, f->h1, (int64_t)B * H, stream))) return rc;
        if ((rc = linear(f, f->h1, H, B, H, f->w.guidance_in1, H, f->e_guid, H, VCB_EPI_BIAS, stream))) return rc;
    }
    if ((rc = linear(f, y, c.vec_in_dim, B, c.vec_in_dim, f->w.vector_in0, H, f->h1, H, VCB_EPI_BIAS, stream))) return rc;
    if ((rc = vcb_silu(f->h1, f->h1, (int64_t)B * H, stream))) return rc;
    if ((rc = linear(f, f->h1, H, B, H, f->w.vector_in1, H, f->e_vec, H, VCB_EPI_BIAS, stream))) return rc;
    if ((rc = vcb_add3(f->e_time, c.guidance_embed ? f->e_guid : nullptr, B, f->e_vec, B, f->vec, EB, H, stream))) return rc;
    if ((rc = vcb_silu(f->vec, f->svec, (int64_t)EB * H, stream))) return rc;
    // AdaLN modulation vectors of all evaluations: one GEMM per block reads each modulation weight once per image
    // instead of once per step (layers.py:121 is a GEMV re-reading 6.5 GB per step in the reference)
    for (int i = 0; i < c.depth; ++i) {
        if ((rc = linear(f, f->svec, H, EB, H, f->dbl[i].img.mod, 6 * H, f->mod_dbl[2 * i], 6 * H, VCB_EPI_BIAS, stream))) return rc;
        if ((rc = linear(f, f->svec, H, EB, H, f->dbl[i].txt.mod, 6 * H, f->mod_dbl[2 * i + 1], 6 * H, VCB_EPI_BIAS, stream))) return rc;
    }
    for (int i = 0; i < c.depth_single; ++i)
        if ((rc = linear(f, f->svec, H, EB, H, f->sgl[i].mod, 3 * H, f->mod_sgl[i], 3 * H, VCB_EPI_BIAS, stream))) return rc;
    if ((rc = linear(f, f->svec, H, EB, H, f->w.final_mod, 2 * H, f->mod_final, 2 * H, VCB_EPI_BIAS, stream))) return rc;
    f->prepared = true;
    return 0;
}

namespace {

struct StreamView {
    int rows;      // tokens of this stream per sample
    int off;       // first row of the stream inside a sample's L rows
};

// GEMM over one stream of the joint buffers: A rows (b, off + i) of `a_buf`, output rows (b, off + i) of `out`
vcb_gemm_args stream_args(const vcb_flux* f, const StreamView& sv, const uint16_t* a_buf, int64_t lda, int a_col, int K,
                          const vcb_linear_w& w, int N, int epi, uint16_t* out, int64_t ldo, int out_col, const uint16_t* gate,
                          int64_t gate_stride, const void* q_scale, const void* k_scale, uint16_t* out2, int64_t ldo2,
                          int out2_col) {
    vcb_gemm_args g{};
    g.M = f->B * sv.rows; g.N = N; g.K = K;
    g.A = a_buf + (int64_t)sv.off * lda + a_col; g.lda = lda; g.a_batch_stride = (int64_t)f->L * lda;
    g.W = w.w; g.ldw = K; g.bias = w.b;
    g.out = out; g.ldo = ldo; g.out_col_offset = out_col;
    g.rows_per_batch = sv.rows; g.out_batch_rows = f->L; g.out_row_offset = sv.off;
    g.epilogue = epi;
    g.gate = gate; g.gate_stride = gate_stride; g.res = out; g.ld_res = ldo;
    // the GEMMs that write the residual stream leave the next LayerNorm's statistics behind (bf16 path; H % 64 == 0 always holds)
    if (epi == VCB_EPI_GATE_RES && out == f->x) g.row_stats = f->row_stats;
    g.hidden = f->cfg.hidden; g.q_scale = q_scale; g.k_scale = k_scale; g.rope = f->rope; g.rope_rows = (int64_t)f->B * f->L;
    g.out2 = out2; g.ldo2 = ldo2; g.out2_col_offset = out2_col;
    if (f->fp8 && a_buf == f->xm && w.w8) {
        // fp8 projection: A = the e4m3 LayerNorm output (same [B, L, H] row layout, one byte per element), W = the e4m3 weight
        g.operand_dtype = VCB_DTYPE_E4M3;
        g.A = f->xm8 + (int64_t)sv.off * lda + a_col;
        g.W = w.w8;
        g.a_scale = f->row_scale; g.w_scale = w.w8_scale;
    } else if (f->fp8 >= 2 && a_buf == f->cat && w.w8) {
        // level 2: A = the e4m3 copy of the cat columns vcb_quantize_rows_e4m3 produced just before (same row layout, bytes)
        g.operand_dtype = VCB_DTYPE_E4M3;
        g.A = f->cat8 + (int64_t)sv.off * lda + a_col;
        g.W = w.w8;
        g.a_scale = f->cat_scale; g.w_scale = w.w8_scale;
    }
    if (f->sp_world > 1 && (epi == VCB_EPI_QKV || epi == VCB_EPI_LINEAR1)) {
        g.sp_world = f->sp_world; g.sp_row_offset = f->sp_rank * f->L;
        for (int r = 0; r < f->sp_world; ++r) g.sp_out[r] = f->sp_qkv[r];
    }
    return g;
}

// attention over the joint sequence; sequence-parallel: barrier, attention of this rank's heads over all ranks' rows with
// the output rows scattered back to their owners, barrier
int joint_attention(vcb_flux* f, int64_t ldc, float score_bound, void* stream) {
    const vcb_flux_config& c = f->cfg;
    const int H = c.hidden;
    vcb_attn_args a{};
    a.score_bound_log2 = f->use_score_bounds ? score_bound : 0.f;
    a.ldo = ldc;
    if (f->sp_world <= 1) {
        a.qkv = f->qkv; a.ld_qkv = 3 * H; a.q_col = 0; a.k_col = H; a.v_col = 2 * H;
        a.seqlens = f->seqlens; a.B = f->B; a.L = f->L; a.heads = c.heads;
        a.out = f->cat; a.out_col_offset = 0;
        return vcb_attention_fwd_ex(&a, stream);
    }
    const int W = f->sp_world, hw = H / W;
    int rc;
    if ((rc = vcb_sp_barrier(f->sp_flags, W, f->sp_rank, ++f->sp_epoch, f->sp_err, f->sp_timeout_ms, stream))) return rc;
    a.qkv = f->qkv; a.ld_qkv = 3 * hw; a.q_col = 0; a.k_col = hw; a.v_col = 2 * hw;
    a.B = 1; a.L = W * f->L; a.heads = c.heads / W;
    a.out_peers = f->sp_cat; a.world = W; a.rows_per_rank = f->L; a.out_col_offset = f->sp_rank * hw;
    if ((rc = vcb_attention_fwd_ex(&a, stream))) return rc;
    return vcb_sp_barrier(f->sp_flags, W, f->sp_rank, ++f->sp_epoch, f->sp_err, f->sp_timeout_ms, stream);
}

// fp8 level 2: e4m3 copy of columns [col0, col0 + K) of every row of `cat` (+ per-row scales) for the Linear that reads them next
int quantize_cat(const vcb_flux* f, int64_t ldc, int col0, int K, void* stream) {
    if (f->fp8 < 2) return 0;
    return vcb_quantize_rows_e4m3(f->cat + col0, ldc, f->cat8 + col0, ldc, f->cat_scale, (int64_t)f->B * f->L, K, stream);
}

int stream_gemm(const vcb_flux* f, const StreamView& sv, const uint16_t* a_buf, int64_t lda, int a_col, int K,
                const vcb_linear_w& w, int N, int epi, uint16_t* out, int64_t ldo, int out_col, const uint16_t* gate,
                int64_t gate_stride, const vcb_stream_w* qk, const void* q_scale, const void* k_scale, uint16_t* out2,
                int64_t ldo2, int out2_col, void* stream) {
    (void)qk;
    vcb_gemm_args g = stream_args(f, sv, a_buf, lda, a_col, K, w, N, epi, out, ldo, out_col, gate, gate_stride, q_scale, k_scale,
                                  out2, ldo2, out2_col);
    return gemm_linear(f, g, w, stream);
}

// The AdaLN LayerNorm of one stream, or of both streams of a DoubleStreamBlock in one launch (sv1 != nullptr).  shift0 / shift1:
// the stream's shift vector; its scale follows at + hidden.
// fp8: the LayerNorm feeds an fp8 projection -> e4m3 rows + per-row scales instead of bf16 rows.
int adaln(const vcb_flux* f, const StreamView& sv0, const uint16_t* shift0, const StreamView* sv1, const uint16_t* shift1, int64_t mod_stride,
          bool fp8, void* stream) {
    const int H = f->cfg.hidden, ns = H / 64;
    const StreamView* sv[2] = {&sv0, sv1};
    const uint16_t* shift[2] = {shift0, shift1};
    vcb_ln_args a[2] = {};
    float* rs[2] = {};
    const float* st[2] = {};
    for (int s = 0; s < (sv1 ? 2 : 1); ++s) {
        const int64_t off = sv[s]->off;
        void* y = fp8 ? (void*)(f->xm8 + off * H) : (void*)(f->xm + off * H);
        a[s] = vcb_ln_args{f->x + off * H, y, shift[s], shift[s] + H, f->B * sv[s]->rows, sv[s]->rows};
        rs[s] = f->row_scale + off;
        st[s] = f->row_stats + off * ns * 2;
    }
    const vcb_ln_args* a1 = sv1 ? &a[1] : nullptr;
    if (f->stats_valid)
        return fp8 ? vcb_ln_modulate_fp8_stats(&a[0], a1, rs[0], rs[1], st[0], st[1], ns, H, H, mod_stride, H, f->L, stream)
                   : vcb_ln_modulate_stats(&a[0], a1, st[0], st[1], ns, H, H, mod_stride, H, f->L, stream);
    return fp8 ? vcb_ln_modulate_fp8(&a[0], a1, rs[0], rs[1], H, H, mod_stride, H, f->L, stream)
               : vcb_ln_modulate_grouped(&a[0], a1, H, H, mod_stride, H, f->L, stream);
}

FbcRows fbc_rows(const vcb_flux* f) { return FbcRows{f->B, f->Li, f->Lt, f->L, f->cfg.hidden, f->seqlens}; }

// First-block cache, right after double block 0: decide (one stream wait, except on the first evaluation since prepare, which is
// always computed), then either write x = bf16(x1 + R) (every group skips) or make r_k the new r_ref and keep x1 for the residual R
// (every group computes).  Per-sample mode with mixed decisions (*mixed): the blocks run for the whole batch; the computed samples'
// rows of r_k become their r_ref, and x1 of every sample is kept for fbc_finish.
int fbc_after_first_block(vcb_flux* f, cudaStream_t st, bool* skip, bool* mixed) {
    const bool first = f->fbc_computed == 0 && f->fbc_skipped == 0;
    const FbcRows g = fbc_rows(f);
    const int groups = f->fbc_per_sample ? f->B : 1;
    uint16_t* x0_rk = f->fbc_buf[f->fbc_ref ^ 1];
    if (int rc = fbc_decide(x0_rk, f->x, f->fbc_buf[f->fbc_ref], g, groups, first, f->fbc_threshold, f->fbc_part, f->fbc_res, st)) return rc;
    *skip = *mixed = false;
    f->fbc_last_diff = INFINITY;
    int n_skip = 0;
    if (!first) {
        cudaError_t e = cudaMemcpyAsync(f->fbc_host, f->fbc_res, (4 * groups + 1) * sizeof(float), cudaMemcpyDeviceToHost, st);
        if (e == cudaSuccess) e = cudaStreamSynchronize(st);
        if (e != cudaSuccess) return set_error("flux_forward: first-block cache decision: %s", cudaGetErrorString(e));
        n_skip = (int)f->fbc_host[4 * groups];
        f->fbc_last_diff = f->fbc_host[2];
    }
    if (f->fbc_per_sample) {
        for (int b = 0; b < f->B; ++b) {
            const bool sb = !first && f->fbc_host[4 * b + 3] != 0.f;
            f->fbc_s_skip[b] = sb;
            f->fbc_s_diff[b] = first ? INFINITY : f->fbc_host[4 * b + 2];
            ++(sb ? f->fbc_s_skipped[b] : f->fbc_s_computed[b]);
            if (b == 0 || f->fbc_s_diff[b] > f->fbc_last_diff) f->fbc_last_diff = f->fbc_s_diff[b];   // the largest sample diff
        }
    }
    const int64_t H = f->cfg.hidden, img_bytes = (int64_t)f->Li * H * 2;
    if (n_skip == groups) {
        *skip = true;
        ++f->fbc_skipped;
        return fbc_apply_residual(f->x, f->fbc_R, g, st);
    }
    ++f->fbc_computed;
    if (n_skip == 0) {
        f->fbc_ref ^= 1;                               // r_k is the reference of the next decisions
    } else {
        *mixed = true;
        for (int b = 0; b < f->B; ++b) {
            if (f->fbc_s_skip[b]) continue;
            cudaError_t e = cudaMemcpyAsync(f->fbc_buf[f->fbc_ref] + b * (int64_t)f->Li * H, x0_rk + b * (int64_t)f->Li * H, (size_t)img_bytes,
                                            cudaMemcpyDeviceToDevice, st);
            if (e != cudaSuccess) return set_error("flux_forward: first-block cache r_ref copy: %s", cudaGetErrorString(e));
        }
    }
    cudaError_t e = cudaMemcpy2DAsync(f->fbc_buf[f->fbc_ref ^ 1], (size_t)img_bytes, f->x + (int64_t)f->Lt * H, (size_t)f->L * H * 2,
                                      (size_t)img_bytes, f->B, cudaMemcpyDeviceToDevice, st);
    if (e != cudaSuccess) return set_error("flux_forward: first-block cache x1 copy: %s", cudaGetErrorString(e));
    return 0;
}

// First-block cache, after the last block of a computed evaluation: R = x_final - x1 for the computed samples; with mixed decisions
// the img rows of each skipped sample become bf16(x1 + R) with its own x1 and R (the same arithmetic as a skipped evaluation)
int fbc_finish(vcb_flux* f, bool mixed, cudaStream_t st) {
    const uint16_t* x1c = f->fbc_buf[f->fbc_ref ^ 1];
    if (!mixed) return fbc_store_residual(f->x, x1c, f->fbc_R, fbc_rows(f), st);
    const int64_t H = f->cfg.hidden, n = (int64_t)f->Li * H;
    const FbcRows one{1, f->Li, f->Lt, f->L, f->cfg.hidden, nullptr};
    for (int b = 0; b < f->B; ++b) {
        uint16_t* xb = f->x + (int64_t)b * f->L * H;
        if (!f->fbc_s_skip[b]) {
            if (int rc = fbc_store_residual(xb, x1c + b * n, f->fbc_R + b * n, one, st)) return rc;
            continue;
        }
        cudaError_t e = cudaMemcpyAsync(xb + (int64_t)f->Lt * H, x1c + b * n, (size_t)n * 2, cudaMemcpyDeviceToDevice, st);
        if (e != cudaSuccess) return set_error("flux_forward: first-block cache x1 restore: %s", cudaGetErrorString(e));
        if (int rc = fbc_apply_residual(xb, f->fbc_R + b * n, one, st)) return rc;
    }
    return 0;
}

}  // namespace

extern "C" int vcb_flux_forward(vcb_flux* f, int32_t e, const void* img, int64_t ld_img, void* out, int64_t ld_out,
                                void* stream) {
    if (!f || !img || !out) return set_error("flux_forward: null argument");
    if (!f->prepared) return set_error("flux_forward: call vcb_flux_prepare first");
    if (e < 0 || e >= f->E) return set_error("flux_forward: eval index %d out of range [0, %d)", e, f->E);
    const vcb_flux_config& c = f->cfg;
    const int H = c.hidden, mlp = c.mlp_hidden, B = f->B, L = f->L, Li = f->Li, Lt = f->Lt;
    const int64_t ldc = H + mlp;
    const StreamView s_img{Li, Lt}, s_txt{Lt, 0}, s_all{L, 0};
    cudaStream_t st = (cudaStream_t)stream;
    int rc;
    // img_in (model.py:101) straight into the img rows of x; txt rows <- txt0
    {
        vcb_gemm_args g{};
        g.M = B * Li; g.N = H; g.K = c.in_channels;
        g.A = img; g.lda = ld_img;
        g.W = f->w.img_in.w; g.ldw = c.in_channels; g.bias = f->w.img_in.b;
        g.out = f->x; g.ldo = H;
        g.rows_per_batch = Li; g.out_batch_rows = L; g.out_row_offset = Lt;
        g.epilogue = VCB_EPI_BIAS;
        if ((rc = gemm_linear(f, g, f->w.img_in, stream))) return rc;
    }
    for (int b = 0; b < B; ++b) {
        cudaError_t ce = cudaMemcpyAsync(f->x + (int64_t)b * L * H, f->txt0 + (int64_t)b * Lt * H, (size_t)Lt * H * 2,
                                         cudaMemcpyDeviceToDevice, st);
        if (ce != cudaSuccess) return set_error("flux_forward: txt copy: %s", cudaGetErrorString(ce));
    }
    f->stats_valid = false;                  // x was just (re)written by img_in and the txt copy: no statistics yet
    const bool fbc = f->fbc_threshold > 0.f;
    bool skip = false, mixed = false;
    if (fbc) {                               // x0: the img rows as img_in left them
        cudaError_t ce = cudaMemcpy2DAsync(f->fbc_buf[f->fbc_ref ^ 1], (size_t)Li * H * 2, f->x + (int64_t)Lt * H, (size_t)L * H * 2,
                                           (size_t)Li * H * 2, B, cudaMemcpyDeviceToDevice, st);
        if (ce != cudaSuccess) return set_error("flux_forward: first-block cache x0 copy: %s", cudaGetErrorString(ce));
    }
    const int64_t erow = (int64_t)e * B;     // first modulation row of this evaluation
    // ---- double-stream blocks (layers.py:158-196) ----
    for (int i = 0; i < c.depth; ++i) {
        const vcb_double_w& w = f->dbl[i];
        const vcb_stream_w* sw[2] = {&w.img, &w.txt};
        const StreamView* sv[2] = {&s_img, &s_txt};
        const uint16_t* mod[2] = {f->mod_dbl[2 * i] + erow * 6 * H, f->mod_dbl[2 * i + 1] + erow * 6 * H};
        // both streams of a block share each launch (img first, txt fills the img problem's partial last wave)
        if ((rc = adaln(f, s_img, mod[0], &s_txt, mod[1], 6 * H, f->fp8, stream))) return rc;
        {
            vcb_gemm_args g[2];
            const vcb_linear_w* lw[2] = {&sw[0]->qkv, &sw[1]->qkv};
            for (int s = 0; s < 2; ++s)
                g[s] = stream_args(f, *sv[s], f->xm, H, 0, H, sw[s]->qkv, 3 * H, VCB_EPI_QKV, f->qkv, 3 * H, 0, nullptr, 0,
                                   sw[s]->q_scale, sw[s]->k_scale, nullptr, 0, 0);
            if ((rc = gemm_linear(f, g, lw, 2, stream))) return rc;
        }
        if ((rc = joint_attention(f, ldc, w.attn_score_bound, stream))) return rc;
        if ((rc = quantize_cat(f, ldc, 0, H, stream))) return rc;
        {
            vcb_gemm_args g[2];
            const vcb_linear_w* lw[2] = {&sw[0]->proj, &sw[1]->proj};
            for (int s = 0; s < 2; ++s)
                g[s] = stream_args(f, *sv[s], f->cat, ldc, 0, H, sw[s]->proj, H, VCB_EPI_GATE_RES, f->x, H, 0, mod[s] + 2 * H, 6 * H,
                                   nullptr, nullptr, nullptr, 0, 0);
            if ((rc = gemm_linear(f, g, lw, 2, stream))) return rc;
            f->stats_valid = true;             // both streams' rows of x now have their LayerNorm statistics in row_stats
        }
        if ((rc = adaln(f, s_img, mod[0] + 3 * H, &s_txt, mod[1] + 3 * H, 6 * H, f->fp8, stream))) return rc;
        {
            vcb_gemm_args g[2];
            const vcb_linear_w* lw[2] = {&sw[0]->mlp0, &sw[1]->mlp0};
            for (int s = 0; s < 2; ++s)
                g[s] = stream_args(f, *sv[s], f->xm, H, 0, H, sw[s]->mlp0, mlp, VCB_EPI_BIAS_GELU, f->cat, ldc, H, nullptr, 0, nullptr,
                                   nullptr, nullptr, 0, 0);
            if ((rc = gemm_linear(f, g, lw, 2, stream))) return rc;
        }
        if ((rc = quantize_cat(f, ldc, H, mlp, stream))) return rc;
        {
            vcb_gemm_args g[2];
            const vcb_linear_w* lw[2] = {&sw[0]->mlp2, &sw[1]->mlp2};
            for (int s = 0; s < 2; ++s)
                g[s] = stream_args(f, *sv[s], f->cat, ldc, H, mlp, sw[s]->mlp2, H, VCB_EPI_GATE_RES, f->x, H, 0, mod[s] + 5 * H, 6 * H,
                                   nullptr, nullptr, nullptr, 0, 0);
            if ((rc = gemm_linear(f, g, lw, 2, stream))) return rc;
            f->stats_valid = true;
        }
        if (i == 0 && fbc) {
            if ((rc = fbc_after_first_block(f, st, &skip, &mixed))) return rc;
            if (skip) break;
        }
    }
    // ---- single-stream blocks on the joint sequence (layers.py:232-245) ----
    for (int i = 0; !skip && i < c.depth_single; ++i) {
        const vcb_single_w& w = f->sgl[i];
        const uint16_t* mod = f->mod_sgl[i] + erow * 3 * H;
        if ((rc = adaln(f, s_all, mod, nullptr, nullptr, 3 * H, f->fp8, stream))) return rc;
        if ((rc = stream_gemm(f, s_all, f->xm, H, 0, H, w.linear1, 3 * H + mlp, VCB_EPI_LINEAR1, f->qkv, 3 * H, 0, nullptr, 0,
                              nullptr, w.q_scale, w.k_scale, f->cat, ldc, H, stream))) return rc;
        if ((rc = joint_attention(f, ldc, w.attn_score_bound, stream))) return rc;
        if ((rc = quantize_cat(f, ldc, 0, H + mlp, stream))) return rc;
        if ((rc = stream_gemm(f, s_all, f->cat, ldc, 0, H + mlp, w.linear2, H, VCB_EPI_GATE_RES, f->x, H, 0, mod + 2 * H, 3 * H,
                              nullptr, nullptr, nullptr, nullptr, 0, 0, stream))) return rc;
        f->stats_valid = true;
    }
    if (fbc) {
        if (!skip && (rc = fbc_finish(f, mixed, st))) return rc;
        // the final LayerNorm computes its own statistics whenever the cache is on: a skipped evaluation (whose x no GEMM
        // epilogue wrote) and a computed one then share the arithmetic, so equal residual streams give equal outputs
        f->stats_valid = false;
    }
    // ---- final layer on the img rows (layers.py:255-259; chunk order shift, scale) ----
    {
        const uint16_t* mod = f->mod_final + erow * 2 * H;
        if ((rc = adaln(f, s_img, mod, nullptr, nullptr, 2 * H, false, stream))) return rc;
        vcb_gemm_args g{};
        g.M = B * Li; g.N = c.out_channels; g.K = H;
        g.A = f->xm + (int64_t)Lt * H; g.lda = H; g.a_batch_stride = (int64_t)L * H;
        g.W = f->w.final_linear.w; g.ldw = H; g.bias = f->w.final_linear.b;
        g.out = out; g.ldo = ld_out;
        g.rows_per_batch = Li; g.out_batch_rows = Li; g.out_row_offset = 0;
        g.epilogue = VCB_EPI_BIAS;
        if ((rc = gemm_linear(f, g, f->w.final_linear, stream))) return rc;
    }
    return 0;
}
