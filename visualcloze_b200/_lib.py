"""ctypes binding of libvcb200.so (include/vcb200.h).  Fails loudly when the library is missing."""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libvcb200.so")
ABI_VERSION = 7
SP_MAX = 8

_lib = None


class VcbError(RuntimeError):
    pass


class GemmArgs(C.Structure):
    """struct vcb_gemm_args (include/vcb200.h)."""
    _fields_ = [
        ("M", C.c_int32), ("N", C.c_int32), ("K", C.c_int32),
        ("A", C.c_void_p), ("lda", C.c_int64), ("a_batch_stride", C.c_int64),
        ("W", C.c_void_p), ("ldw", C.c_int64),
        ("bias", C.c_void_p),
        ("out", C.c_void_p), ("ldo", C.c_int64),
        ("out_col_offset", C.c_int32),
        ("rows_per_batch", C.c_int32), ("out_batch_rows", C.c_int32), ("out_row_offset", C.c_int32),
        ("epilogue", C.c_int32),
        ("gate", C.c_void_p), ("gate_stride", C.c_int64),
        ("res", C.c_void_p), ("ld_res", C.c_int64),
        ("hidden", C.c_int32),
        ("q_scale", C.c_void_p), ("k_scale", C.c_void_p),
        ("rope", C.c_void_p), ("rope_rows", C.c_int64),
        ("out2", C.c_void_p), ("ldo2", C.c_int64), ("out2_col_offset", C.c_int32),
        ("block_n", C.c_int32), ("cta_group", C.c_int32),
        ("sp_world", C.c_int32), ("sp_row_offset", C.c_int32), ("sp_out", C.c_void_p * SP_MAX),
        ("row_stats", C.c_void_p),
        ("operand_dtype", C.c_int32), ("a_scale", C.c_void_p), ("w_scale", C.c_void_p),
        ("lora_t", C.c_void_p), ("ld_lora_t", C.c_int64), ("lora_t_batch_stride", C.c_int64), ("lora_b", C.c_void_p),
        ("lora_rank", C.c_int32), ("alpha", C.c_float),
    ]


_SIGNATURES = {
    "vcb_abi_version": (C.c_int, []),
    "vcb_last_error": (C.c_char_p, []),
    "vcb_launch_count": (C.c_longlong, []),
    "vcb_reset_launch_count": (None, []),
    "vcb_debug_attn4_timeline": (C.c_int, [C.c_void_p, C.c_int32]),
    "vcb_profile_begin": (C.c_int, []),
    "vcb_profile_end": (C.c_int, [C.POINTER(C.c_double), C.POINTER(C.c_longlong)]),
    "vcb_profile_end_ex": (C.c_int, [C.POINTER(C.c_double), C.POINTER(C.c_longlong), C.c_int32, C.c_void_p, C.c_int64,
                                     C.POINTER(C.c_int64)]),
    "vcb_gemm_bf16": (C.c_int, [C.POINTER(GemmArgs), C.c_void_p]),
    "vcb_gemm_bf16_grouped": (C.c_int, [C.POINTER(GemmArgs), C.POINTER(GemmArgs), C.c_void_p]),
    "vcb_conv3x3_nhwc": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32,
                                   C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p]),
    "vcb_attention_fwd": (C.c_int, [C.c_void_p, C.c_int64, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_int32,
                                    C.c_int32, C.c_int32, C.c_void_p, C.c_int64, C.c_int32, C.c_void_p]),
    "vcb_ln_modulate": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_int64,
                                  C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p]),
    "vcb_timestep_embedding": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p]),
    "vcb_silu": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]),
    "vcb_embedding_bf16": (C.c_int, [C.c_void_p, C.c_int64, C.c_int32, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_int64, C.c_int64, C.c_void_p]),
    "vcb_rmsnorm_weight": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_int32, C.c_float, C.c_void_p]),
    "vcb_layernorm_affine": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_int32, C.c_float, C.c_void_p]),
    "vcb_gated_gelu": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_int64, C.c_int32, C.c_void_p]),
    "vcb_quick_gelu": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]),
    "vcb_add3": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32,
                           C.c_int32, C.c_void_p]),
    "vcb_rope_table": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_double,
                                 C.c_void_p]),
    "vcb_euler_update": (C.c_int, [C.c_void_p, C.c_void_p, C.c_float, C.c_void_p, C.c_void_p, C.c_int64, C.c_int64,
                                   C.c_int32, C.c_void_p]),
    "vcb_ode_stage": (C.c_int, [C.c_int32, C.c_int32, C.c_void_p, C.POINTER(C.c_void_p), C.c_int32, C.c_float, C.c_void_p,
                                C.c_void_p, C.c_int64, C.c_int64, C.c_int32, C.c_void_p]),
    "vcb_copy_cols": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_int32, C.c_int64, C.c_int32,
                                C.c_void_p]),
    "vcb_debug_umma_probe": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32,
                                       C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p]),
}

class LinearW(C.Structure):
    """struct vcb_linear_w (include/vcb200.h): rank 0 = merged weight, rank > 0 = unmerged LoRA (w, lora_a, lora_b, lora_scale)."""
    _fields_ = [("w", C.c_void_p), ("b", C.c_void_p), ("w8", C.c_void_p), ("w8_scale", C.c_void_p),
                ("lora_a", C.c_void_p), ("lora_b", C.c_void_p), ("rank", C.c_int32), ("lora_scale", C.c_float)]


class StreamW(C.Structure):
    _fields_ = [("mod", LinearW), ("qkv", LinearW), ("proj", LinearW), ("mlp0", LinearW), ("mlp2", LinearW),
                ("q_scale", C.c_void_p), ("k_scale", C.c_void_p)]


class DoubleW(C.Structure):
    _fields_ = [("img", StreamW), ("txt", StreamW), ("attn_score_bound", C.c_float)]


class SingleW(C.Structure):
    _fields_ = [("mod", LinearW), ("linear1", LinearW), ("linear2", LinearW), ("q_scale", C.c_void_p),
                ("k_scale", C.c_void_p), ("attn_score_bound", C.c_float)]


class LnArgs(C.Structure):
    """struct vcb_ln_args (include/vcb200.h)."""
    _fields_ = [("x", C.c_void_p), ("y", C.c_void_p), ("shift", C.c_void_p), ("scale", C.c_void_p), ("rows", C.c_int32),
                ("rows_per_batch", C.c_int32)]


class AttnArgs(C.Structure):
    """struct vcb_attn_args (include/vcb200.h)."""
    _fields_ = [("qkv", C.c_void_p), ("ld_qkv", C.c_int64), ("q_col", C.c_int32), ("k_col", C.c_int32), ("v_col", C.c_int32),
                ("seqlens", C.c_void_p), ("B", C.c_int32), ("L", C.c_int32), ("heads", C.c_int32),
                ("out", C.c_void_p), ("ldo", C.c_int64), ("out_col_offset", C.c_int32),
                ("out_peers", C.POINTER(C.c_void_p)), ("world", C.c_int32), ("rows_per_rank", C.c_int32),
                ("score_bound_log2", C.c_float), ("schedule", C.c_int32)]


class AttnSmallArgs(C.Structure):
    """struct vcb_attn_small_args (include/vcb200.h)."""
    _fields_ = [("q", C.c_void_p), ("k", C.c_void_p), ("v", C.c_void_p), ("ld", C.c_int64), ("bias", C.c_void_p),
                ("out", C.c_void_p), ("ldo", C.c_int64), ("B", C.c_int32), ("L", C.c_int32), ("heads", C.c_int32),
                ("head_dim", C.c_int32), ("causal", C.c_int32), ("scale", C.c_float)]


class ProfRecord(C.Structure):
    """struct vcb_prof_record (include/vcb200.h)."""
    _fields_ = [("category", C.c_int32), ("ms", C.c_float), ("info", C.c_int32 * 4)]


PROF_CATEGORIES = ("gemm", "attention", "ln_modulate", "other", "vae_conv3x3", "vae_elementwise")


def profile_end(max_records: int = 0):
    """-> ({category: (ms, launches)}, [ProfRecord...]) for everything launched since vcb_profile_begin (synchronises)."""
    ms, n = (C.c_double * 6)(), (C.c_longlong * 6)()
    recs = (ProfRecord * max_records)() if max_records else None
    cnt = C.c_int64(0)
    check(lib().vcb_profile_end_ex(ms, n, 6, C.cast(recs, C.c_void_p) if recs is not None else None, max_records, C.byref(cnt)),
          "vcb_profile_end_ex")
    out = {name: (ms[i], int(n[i])) for i, name in enumerate(PROF_CATEGORIES)}
    return out, ([] if recs is None else list(recs[:min(int(cnt.value), max_records)]))


class FluxConfigC(C.Structure):
    _fields_ = [("in_channels", C.c_int32), ("out_channels", C.c_int32), ("vec_in_dim", C.c_int32),
                ("context_in_dim", C.c_int32), ("hidden", C.c_int32), ("mlp_hidden", C.c_int32), ("heads", C.c_int32),
                ("depth", C.c_int32), ("depth_single", C.c_int32), ("axes_dim", C.c_int32 * 3),
                ("guidance_embed", C.c_int32), ("theta", C.c_double)]


class FluxWeightsC(C.Structure):
    _fields_ = [("img_in", LinearW), ("txt_in", LinearW), ("time_in0", LinearW), ("time_in1", LinearW),
                ("vector_in0", LinearW), ("vector_in1", LinearW), ("guidance_in0", LinearW), ("guidance_in1", LinearW),
                ("final_mod", LinearW), ("final_linear", LinearW),
                ("dbl", C.POINTER(DoubleW)), ("sgl", C.POINTER(SingleW))]


class ConvW(C.Structure):
    _fields_ = [("w", C.c_void_p), ("b", C.c_void_p), ("cin", C.c_int32), ("cout", C.c_int32)]


class GnW(C.Structure):
    _fields_ = [("gamma", C.c_void_p), ("beta", C.c_void_p)]


class ResblockW(C.Structure):
    _fields_ = [("norm1", GnW), ("conv1", ConvW), ("norm2", GnW), ("conv2", ConvW), ("shortcut", ConvW)]


class VaeConfigC(C.Structure):
    _fields_ = [("ch", C.c_int32), ("out_ch", C.c_int32), ("z_channels", C.c_int32), ("num_res_blocks", C.c_int32),
                ("n_levels", C.c_int32), ("ch_mult", C.c_int32 * 8), ("scale_factor", C.c_float), ("shift_factor", C.c_float)]


class VaeWeightsC(C.Structure):
    _fields_ = [("conv_in", ConvW), ("mid1", ResblockW), ("mid2", ResblockW), ("attn_norm", GnW),
                ("attn_q", ConvW), ("attn_k", ConvW), ("attn_v", ConvW), ("attn_proj", ConvW),
                ("up_blocks", C.POINTER(ResblockW)), ("upsample", C.POINTER(ConvW)), ("norm_out", GnW), ("conv_out", ConvW)]


class VaeEncWeightsC(C.Structure):
    _fields_ = [("conv_in", ConvW), ("down_blocks", C.POINTER(ResblockW)), ("downsample", C.POINTER(ConvW)),
                ("mid1", ResblockW), ("mid2", ResblockW), ("attn_norm", GnW),
                ("attn_q", ConvW), ("attn_k", ConvW), ("attn_v", ConvW), ("attn_proj", ConvW),
                ("norm_out", GnW), ("conv_out", ConvW)]


_OPTIONAL: dict = {
    "vcb_vae_enc_create": (C.c_int, [C.POINTER(VaeConfigC), C.POINTER(VaeEncWeightsC), C.POINTER(C.c_void_p)]),
    "vcb_vae_enc_destroy": (None, [C.c_void_p]),
    "vcb_vae_enc_workspace_bytes": (C.c_int64, [C.c_void_p, C.c_int32, C.c_int32, C.c_int32]),
    "vcb_vae_encode": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_int32, C.c_int32, C.c_int32,
                                 C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "vcb_vae_create": (C.c_int, [C.POINTER(VaeConfigC), C.POINTER(VaeWeightsC), C.POINTER(C.c_void_p)]),
    "vcb_vae_destroy": (None, [C.c_void_p]),
    "vcb_vae_workspace_bytes": (C.c_int64, [C.c_void_p, C.c_int32, C.c_int32, C.c_int32]),
    "vcb_vae_decode": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_int32, C.c_int32, C.c_int32,
                                 C.c_void_p, C.c_void_p, C.c_void_p]),
    "vcb_flux_create": (C.c_int, [C.POINTER(FluxConfigC), C.POINTER(FluxWeightsC), C.POINTER(C.c_void_p)]),
    "vcb_flux_destroy": (None, [C.c_void_p]),
    "vcb_flux_use_score_bounds": (C.c_int, [C.c_void_p, C.c_int32]),
    "vcb_flux_set_fp8": (C.c_int, [C.c_void_p, C.c_int32]),
    "vcb_quantize_rows_e4m3": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_int32, C.c_void_p]),
    "vcb_flux_workspace_bytes": (C.c_int64, [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32]),
    "vcb_flux_prepare": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                   C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                   C.c_void_p]),
    "vcb_flux_forward": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p]),
    "vcb_flux_set_first_block_cache": (C.c_int, [C.c_void_p, C.c_float]),
    "vcb_flux_cache_stats": (C.c_int, [C.c_void_p, C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.POINTER(C.c_float)]),
    # sequence-parallel single-image mode
    "vcb_attention_fwd_sp": (C.c_int, [C.c_void_p, C.c_int64, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                       C.POINTER(C.c_void_p), C.c_int32, C.c_int32, C.c_int64, C.c_int32, C.c_void_p]),
    "vcb_attention_fwd_ex": (C.c_int, [C.POINTER(AttnArgs), C.c_void_p]),
    "vcb_attention_small": (C.c_int, [C.POINTER(AttnSmallArgs), C.c_void_p]),
    "vcb_ln_modulate_grouped": (C.c_int, [C.POINTER(LnArgs), C.POINTER(LnArgs), C.c_int64, C.c_int64, C.c_int64, C.c_int32,
                                          C.c_int32, C.c_void_p]),
    "vcb_ln_modulate_stats": (C.c_int, [C.POINTER(LnArgs), C.POINTER(LnArgs), C.c_void_p, C.c_void_p, C.c_int32, C.c_int64, C.c_int64,
                                        C.c_int64, C.c_int32, C.c_int32, C.c_void_p]),
    "vcb_ln_modulate_fp8_stats": (C.c_int, [C.POINTER(LnArgs), C.POINTER(LnArgs), C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32,
                                            C.c_int64, C.c_int64, C.c_int64, C.c_int32, C.c_int32, C.c_void_p]),
    "vcb_ln_modulate_fp8": (C.c_int, [C.POINTER(LnArgs), C.POINTER(LnArgs), C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_int64,
                                      C.c_int32, C.c_int32, C.c_void_p]),
    "vcb_peer_alloc": (C.c_int, [C.c_int64, C.POINTER(C.c_void_p), C.c_void_p]),
    "vcb_peer_open": (C.c_int, [C.c_void_p, C.POINTER(C.c_void_p)]),
    "vcb_peer_close": (C.c_int, [C.c_void_p]),
    "vcb_peer_free": (C.c_int, [C.c_void_p]),
    "vcb_sp_barrier": (C.c_int, [C.POINTER(C.c_void_p), C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p]),
    "vcb_flux_sp_shared_bytes": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.POINTER(C.c_int64), C.POINTER(C.c_int64)]),
    "vcb_flux_sp_attach": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.POINTER(C.c_void_p), C.POINTER(C.c_void_p),
                                     C.POINTER(C.c_void_p), C.c_void_p, C.c_int32]),
}


def exported_symbols() -> list[str]:
    return list(_SIGNATURES) + list(_OPTIONAL)


def lib() -> C.CDLL:
    """Load (once) and return the library; raises VcbError if it has not been built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise VcbError(
                f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                "(visualcloze_b200/csrc/build.sh).  There is no CPU / PyTorch fallback for this path.")
        l = C.CDLL(LIB_PATH)
        for name, (res, args) in {**_SIGNATURES, **_OPTIONAL}.items():
            fn = getattr(l, name)
            fn.restype = res
            fn.argtypes = args
        if l.vcb_abi_version() != ABI_VERSION:
            raise VcbError(f"libvcb200.so ABI {l.vcb_abi_version()} != binding ABI {ABI_VERSION}; rebuild")
        _lib = l
    return _lib


def check(rc: int, what: str = "") -> None:
    if rc != 0:
        msg = lib().vcb_last_error()
        raise VcbError(f"{what}: {msg.decode() if msg else 'error ' + str(rc)}")
