"""Host-side driver of the FLUX-DiT engine in libvcb200 (vcb_flux_* in include/vcb200.h).

Packs the reference's parameters, owns the device workspace, and marshals pointers.  LoRA is either merged (``W + s * B @ A``
formed once at packing time, a second copy of the weights) or unmerged (the engine points at the module's own ``W``, ``A``
and ``B``; every call adds ``s * (x A^T) B^T`` in the GEMM's k-tail).  Arithmetic done here in torch is limited to that one-off
packing and scalar/host bookkeeping (time grids, masks -> sequence lengths); every per-token operation of the path runs in
the library.
"""
from __future__ import annotations

import ctypes as C
import math

import torch
from torch import Tensor

from . import _lib
from ._lib import DoubleW, FluxConfigC, FluxWeightsC, LinearW, SingleW, StreamW, check

BF16 = torch.bfloat16


def first_block_cache_threshold(threshold) -> float:
    """Validated threshold of the first-block cache: None or 0 = off, else a finite number > 0."""
    if threshold is None:
        return 0.0
    if isinstance(threshold, bool) or not isinstance(threshold, (int, float)):
        raise ValueError(f"first-block cache threshold must be a number or None, got {threshold!r}")
    t = float(threshold)
    if not math.isfinite(t) or t < 0:
        raise ValueError(f"first-block cache threshold must be finite and >= 0 (0 or None = off), got {threshold!r}")
    return t


def _freqs() -> Tensor:
    """frequency table of timestep_embedding (layers.py:39), computed exactly like the reference does."""
    half = 128
    return torch.exp(-math.log(10000) * torch.arange(start=0, end=half, dtype=torch.float32) / half)


class FluxEngine:
    def __init__(self, params, named_params: dict[str, Tensor], lora_scale: float = 1.0, fp8: int = 0, lora_mode: str = "merged",
                 workspace: Tensor | None = None):
        """``lora_mode``: "merged" or "unmerged" (see the module docstring; unmerged takes bf16 projections only).
        ``workspace``: a previous engine's device workspace to reuse (grown on demand by ``prepare``)."""
        if lora_mode not in ("merged", "unmerged"):
            raise ValueError("lora_mode must be 'merged' or 'unmerged'")
        if lora_mode == "unmerged" and fp8:
            raise ValueError("unmerged LoRA runs on bf16 operands; the fp8 projections need merged weights")
        some = next(iter(named_params.values()))
        if not some.is_cuda:
            raise _lib.VcbError("FluxEngine needs the model on a CUDA device: the hot path has no CPU fallback")
        self.params = params
        self.device = some.device
        self.lib = _lib.lib()
        self._keep: list[Tensor] = []          # packed tensors referenced by the C structs
        self._p = named_params
        self._scale = float(lora_scale)
        self.fp8 = int(fp8)                    # 0 = bf16, 1 = LayerNorm-fed Linears on e4m3, 2 = every block Linear on e4m3
        self.lora_mode = lora_mode
        self.H = params.hidden_size
        self.mlp = int(params.hidden_size * params.mlp_ratio)
        with torch.no_grad():
            self._build()
        self._ws = workspace
        self._shape = None
        self._sp = None
        self._fbc = 0.0
        self._fbc_per_sample = False
        self._freqs = _freqs().to(self.device)

    # ---- single-image sequence parallelism (SURVEY.md 8f-2) -------------------------------------------
    def enable_sequence_parallel(self, sp) -> None:
        """``sp``: a ``parallel.SequenceParallel`` (or None to switch back).  Every rank then passes the FULL txt / ids to
        ``prepare`` (identical on all ranks) and its LOCAL img rows (``sp.shard``) to ``forward``."""
        if sp is not None and sp.world > 1 and self.lora_mode == "unmerged":
            raise ValueError("sequence-parallel mode takes merged LoRA weights only")
        if sp is not None and sp.world > 1 and self._fbc > 0:
            raise ValueError("the first-block cache decides per batch on one GPU; switch it off before sequence parallelism")
        if sp is not None and self.params.num_heads % sp.world:
            raise ValueError(f"num_heads ({self.params.num_heads}) must be a multiple of the sequence-parallel world size ({sp.world})")
        if sp is None and self._sp is not None:
            check(self.lib.vcb_flux_sp_attach(self._h, 1, 0, None, None, None, None, 0), "vcb_flux_sp_attach")
            self._sp.release()
        self._sp = sp if (sp is not None and sp.world > 1) else None
        self._shape = None

    # ---- first-block cache (vcb_flux_set_first_block_cache) ------------------------------------------
    def set_first_block_cache(self, threshold, per_sample: bool = False) -> None:
        """``threshold`` > 0: an evaluation whose double-block-0 residual moved by less than ``threshold`` (relative L1) since the
        last computed evaluation reuses that evaluation's residual of the remaining blocks; 0 / None: off.  ``per_sample``: one
        decision per sample instead of one per batch (vcb_flux_set_first_block_cache_ex).  Each ``forward`` then waits for its
        decision on the host (not capturable in a CUDA graph)."""
        t = first_block_cache_threshold(threshold)
        per_sample = bool(per_sample)
        if t > 0 and self._sp is not None:
            raise ValueError("the first-block cache decides per batch on one GPU; it is refused with sequence parallelism")
        check(self.lib.vcb_flux_set_first_block_cache_ex(self._h, t, int(per_sample)), "vcb_flux_set_first_block_cache_ex")
        if (t > 0) != (self._fbc > 0) or (t > 0 and per_sample != self._fbc_per_sample):
            self._shape = None                 # the workspace layout changed: prepare again
        self._fbc, self._fbc_per_sample = t, per_sample

    def cache_stats(self) -> dict:
        """{"computed", "skipped"}: evaluations since the last ``prepare``; "last_diff": the latest evaluation's relative change of
        the first-block residual (inf for the first after ``prepare``, NaN before any)."""
        c, s, d = C.c_int32(), C.c_int32(), C.c_float()
        check(self.lib.vcb_flux_cache_stats(self._h, C.byref(c), C.byref(s), C.byref(d)), "vcb_flux_cache_stats")
        return {"computed": int(c.value), "skipped": int(s.value), "last_diff": float(d.value)}

    def sample_cache_stats(self) -> list[dict]:
        """``cache_stats`` of every sample of the prepared batch: its own counters in per-sample mode, the batch's otherwise."""
        if self._shape is None:
            raise _lib.VcbError("FluxEngine.sample_cache_stats called before prepare")
        B = self._shape[0]
        c, s, d = (C.c_int32 * B)(), (C.c_int32 * B)(), (C.c_float * B)()
        check(self.lib.vcb_flux_cache_stats_per_sample(self._h, B, c, s, d), "vcb_flux_cache_stats_per_sample")
        return [{"computed": int(c[b]), "skipped": int(s[b]), "last_diff": float(d[b])} for b in range(B)]

    # ---- weight packing -----------------------------------------------------------------------
    def _linear(self, name: str, fp8: bool = False) -> LinearW:
        """``fp8``: also keep an e4m3 copy of the merged weight with one fp32 scale per output channel (amax / 448) for the
        opt-in fp8 projections (quantised from the fp32 merged weight, not from its bf16 rounding)."""
        p = self._p
        w = p[name + ".weight"]
        a = p.get(name + ".lora_A.weight")
        b = p.get(name + ".bias")
        if self.lora_mode == "unmerged":
            return self._linear_unmerged(name, w, a, b)
        w32 = None
        if a is not None:
            # merged LoRA (lora.py:92-98): W' = W + s * B A in fp32, rounded once to bf16
            w32 = w.float() + self._scale * (p[name + ".lora_B.weight"].float() @ a.float())
            w = w32.to(BF16)
        else:
            w = w.to(BF16)
        w = w.contiguous()
        w8 = w8s = None
        if fp8:
            w32 = w.float() if w32 is None else w32
            w8s = (w32.abs().amax(dim=1).clamp_min(1e-12) / 448.0).contiguous()
            w8 = (w32 / w8s[:, None]).to(torch.float8_e4m3fn).contiguous()
            self._keep += [w8, w8s]
        del w32
        bias = self._bias(name, b, w.shape[0])
        self._keep.append(w)
        return LinearW(w.data_ptr(), bias.data_ptr(), 0 if w8 is None else w8.data_ptr(), 0 if w8s is None else w8s.data_ptr())

    def _bias(self, name: str, b: Tensor | None, n: int) -> Tensor:
        """fp32 bias of the packed Linear: ``b + s * b_B`` (lora.py:92-98)."""
        bias = torch.zeros(n, dtype=torch.float32, device=self.device) if b is None else b.float()
        bb = self._p.get(name + ".lora_B.bias")
        if bb is not None:
            bias = bias + self._scale * bb.float()
        bias = bias.contiguous()
        self._keep.append(bias)
        return bias

    def _linear_unmerged(self, name: str, w: Tensor, a: Tensor | None, b: Tensor | None) -> LinearW:
        """Unmerged LoRA: the module's own bf16 ``weight``, ``lora_A`` [r, in] and ``lora_B`` [out, r] (no copy when they are bf16
        and contiguous, as FluxLoraWrapper's parameters are); only the fp32 bias ``b + s * b_B`` is formed here."""
        w = w.to(BF16).contiguous()
        self._keep.append(w)
        bias = self._bias(name, b, w.shape[0])
        if a is None:
            return LinearW(w.data_ptr(), bias.data_ptr(), 0, 0, 0, 0, 0, 0.0)
        a = a.to(BF16).contiguous()
        lb = self._p[name + ".lora_B.weight"].to(BF16).contiguous()
        self._keep += [a, lb]
        return LinearW(w.data_ptr(), bias.data_ptr(), 0, 0, a.data_ptr(), lb.data_ptr(), a.shape[0], self._scale)

    def _scale_vec(self, name: str) -> int:
        t = self._p[name].to(BF16).contiguous()
        self._keep.append(t)
        return t.data_ptr()

    def _score_bound(self, q_names: list[str], k_names: list[str]) -> float:
        """Upper bound (log2 units) of the scaled attention scores of a block, from its QK-norm scales: after RMSNorm
        ``|q| <= max|q_scale| * sqrt(128)`` (RoPE is a rotation), so ``|q.k| * 128^-0.5 <= max|qs| * max|ks| * sqrt(128)``;
        3 % margin for the bf16 roundings.  0 (= exact online softmax in the kernel) when the bound leaves the safe
        exponent range (b > 48).  One-off host arithmetic on 128-element vectors at weight-packing time."""
        qs = max(float(self._p[n].float().abs().max()) for n in q_names)
        ks = max(float(self._p[n].float().abs().max()) for n in k_names)
        b = qs * ks * math.sqrt(128.0) * math.log2(math.e) * 1.03
        # exp2(s - b) >= 2^-(2b / 1.03): b <= 48 keeps even an all-anti-aligned row ~2^30 above the fp32 / bf16 underflow threshold
        return b if 0.0 < b <= 48.0 else 0.0

    def _build(self):
        P = self.params
        cfg = FluxConfigC()
        cfg.in_channels, cfg.out_channels = P.in_channels, P.out_channels
        cfg.vec_in_dim, cfg.context_in_dim = P.vec_in_dim, P.context_in_dim
        cfg.hidden, cfg.mlp_hidden, cfg.heads = self.H, self.mlp, P.num_heads
        cfg.depth, cfg.depth_single = P.depth, P.depth_single_blocks
        cfg.axes_dim[0], cfg.axes_dim[1], cfg.axes_dim[2] = P.axes_dim
        cfg.guidance_embed, cfg.theta = int(P.guidance_embed), float(P.theta)
        w = FluxWeightsC()
        w.img_in, w.txt_in = self._linear("img_in"), self._linear("txt_in")
        w.time_in0, w.time_in1 = self._linear("time_in.in_layer"), self._linear("time_in.out_layer")
        w.vector_in0, w.vector_in1 = self._linear("vector_in.in_layer"), self._linear("vector_in.out_layer")
        if P.guidance_embed:
            w.guidance_in0, w.guidance_in1 = self._linear("guidance_in.in_layer"), self._linear("guidance_in.out_layer")
        w.final_mod, w.final_linear = self._linear("final_layer.adaLN_modulation.1"), self._linear("final_layer.linear")
        dbl = (DoubleW * max(1, P.depth))()
        for i in range(P.depth):
            for s, dst in (("img", dbl[i].img), ("txt", dbl[i].txt)):
                b = f"double_blocks.{i}.{s}"
                dst.mod, dst.qkv, dst.proj = self._linear(b + "_mod.lin"), self._linear(b + "_attn.qkv", self.fp8 >= 1), self._linear(b + "_attn.proj", self.fp8 >= 2)
                dst.mlp0, dst.mlp2 = self._linear(b + "_mlp.0", self.fp8 >= 1), self._linear(b + "_mlp.2", self.fp8 >= 2)
                dst.q_scale = self._scale_vec(b + "_attn.norm.query_norm.scale")
                dst.k_scale = self._scale_vec(b + "_attn.norm.key_norm.scale")
            dbl[i].attn_score_bound = self._score_bound(
                [f"double_blocks.{i}.{s}_attn.norm.query_norm.scale" for s in ("img", "txt")],
                [f"double_blocks.{i}.{s}_attn.norm.key_norm.scale" for s in ("img", "txt")])
        sgl = (SingleW * max(1, P.depth_single_blocks))()
        for i in range(P.depth_single_blocks):
            b = f"single_blocks.{i}"
            sgl[i].mod, sgl[i].linear1, sgl[i].linear2 = self._linear(b + ".modulation.lin"), self._linear(b + ".linear1", self.fp8 >= 1), self._linear(b + ".linear2", self.fp8 >= 2)
            sgl[i].q_scale = self._scale_vec(b + ".norm.query_norm.scale")
            sgl[i].k_scale = self._scale_vec(b + ".norm.key_norm.scale")
            sgl[i].attn_score_bound = self._score_bound([b + ".norm.query_norm.scale"], [b + ".norm.key_norm.scale"])
        w.dbl, w.sgl = C.cast(dbl, C.POINTER(DoubleW)), C.cast(sgl, C.POINTER(SingleW))
        self._cfg, self._w, self._dbl, self._sgl = cfg, w, dbl, sgl
        h = C.c_void_p()
        check(self.lib.vcb_flux_create(C.byref(cfg), C.byref(w), C.byref(h)), "vcb_flux_create")
        self._h = h
        if self.fp8:
            check(self.lib.vcb_flux_set_fp8(h, self.fp8), "vcb_flux_set_fp8")

    def use_score_bounds(self, enable: bool) -> None:
        """False: every block runs the exact online-max softmax kernel (what a checkpoint whose QK-norm scales leave the safe
        range gets anyway); True (default): blocks with a packed bound use the fixed-reference softmax."""
        check(self.lib.vcb_flux_use_score_bounds(self._h, int(bool(enable))), "vcb_flux_use_score_bounds")

    def softmax_variants(self) -> dict:
        """how many blocks carry a usable score bound (-> fixed-reference softmax) vs none (-> exact online max)"""
        b = [self._dbl[i].attn_score_bound for i in range(self.params.depth)] + \
            [self._sgl[i].attn_score_bound for i in range(self.params.depth_single_blocks)]
        return {"fixed_reference": sum(1 for v in b if v > 0), "exact_online_max": sum(1 for v in b if not v > 0),
                "max_bound_log2": max(b) if b else 0.0}

    def __del__(self):
        h = getattr(self, "_h", None)
        if h:
            self.lib.vcb_flux_destroy(h)
            self._h = None

    # ---- per-image state ------------------------------------------------------------------------
    def prepare(self, *, txt: Tensor, y: Tensor, img_ids: Tensor, txt_ids: Tensor, timesteps: Tensor,
                guidance: Tensor | None, txt_mask: Tensor | None, img_mask: Tensor | None, n_img_tokens: int) -> None:
        """Step-invariant work for ``E = timesteps.shape[0]`` evaluations (timesteps [E, B], FLUX time)."""
        if txt.ndim != 3:
            raise ValueError("Input img and txt tensors must have 3 dimensions.")
        B, Lt, _ = txt.shape
        Li = int(n_img_tokens)
        E = int(timesteps.shape[0])
        dev = self.device
        st = torch.cuda.current_stream().cuda_stream
        sp = self._sp
        if sp is not None:
            # one unpadded sample, rows of both streams split evenly over the ranks; ``n_img_tokens`` is the FULL count
            if B != 1:
                raise ValueError("sequence-parallel mode shares ONE sample across the ranks (batch must be 1)")
            for m in (txt_mask, img_mask):
                if m is not None and not bool(m.to(torch.bool).all()):
                    raise ValueError("sequence-parallel mode does not take padded samples")
            txt_mask = img_mask = None
            txt, txt_ids, img_ids = sp.shard(txt), sp.shard(txt_ids), sp.shard(img_ids)
            Lt, Li = txt.shape[1], sp.row_slice(Li).stop - sp.row_slice(Li).start
            sp.attach(self, Li, Lt)
        need = self.lib.vcb_flux_workspace_bytes(self._h, B, Li, Lt, E)
        if need < 0:
            raise _lib.VcbError("vcb_flux_workspace_bytes: bad shape")
        if self._ws is None or self._ws.numel() < need:
            self._ws = torch.empty(int(need), dtype=torch.uint8, device=dev)
        # `time_factor * t` in the dtype the reference computes it in (layers.py:37): fp32 timesteps stay fp32,
        # the bf16 guidance is scaled in bf16 (30 -> 29952, SURVEY.md appendix A)
        ts = (1000.0 * timesteps.to(dev)).float().reshape(E * B).contiguous()
        gs = None
        if self.params.guidance_embed:
            if guidance is None:
                raise ValueError("Didn't get guidance strength for guidance distilled model.")
            gs = (1000.0 * guidance.to(dev)).float().reshape(B).contiguous()
        ids = torch.cat((txt_ids.to(dev), img_ids.to(dev)), dim=1).float().contiguous()
        if ids.shape != (B, Lt + Li, 3):
            raise ValueError(f"ids must be [B, Lt+Li, 3], got {tuple(ids.shape)}")
        # Masks -> per-sample valid length of the joint [txt | img] sequence.  The kernels treat the FIRST seqlen rows as valid
        # (the layout the pipeline produces: txt_mask all ones, sampling.py:98; img right-padded to the batch max, :82-88).
        # The reference's _upad_input honours arbitrary masks (math.py:40-60); anything else is refused here rather than
        # silently attending to padded txt rows (one host sync per image, where the reference has two per attention call).
        seqlens = None
        if txt_mask is not None or img_mask is not None:
            tm = (txt_mask.to(dev) != 0) if txt_mask is not None else torch.ones(B, Lt, dtype=torch.bool, device=dev)
            im = (img_mask.to(dev) != 0) if img_mask is not None else torch.ones(B, Li, dtype=torch.bool, device=dev)
            if tuple(tm.shape) != (B, Lt) or tuple(im.shape) != (B, Li):
                raise ValueError(f"txt_mask / img_mask must be [B, Lt] / [B, Li] = {(B, Lt)} / {(B, Li)}")
            n_img = im.sum(dim=-1, dtype=torch.int32)
            prefix = torch.arange(Li, device=dev)[None, :] < n_img[:, None]
            if not bool(tm.all() & (im == prefix).all()):
                raise ValueError("unsupported attention mask: the sm_90a attention kernel takes a fully valid txt_mask and a "
                                 "right-padded (prefix) img_mask -- the layout prepare_modified produces (models/sampling.py:82-98)")
            if img_mask is not None:
                seqlens = (n_img + Lt).contiguous()
        txt_c = txt.to(dev, BF16).contiguous()
        y_c = y.to(dev, BF16).contiguous()
        self._hold = (ts, gs, ids, seqlens, txt_c, y_c)      # keep alive until the next prepare
        check(self.lib.vcb_flux_prepare(self._h, self._ws.data_ptr(), self._ws.numel(), B, Li, Lt, E, txt_c.data_ptr(),
                                        y_c.data_ptr(), ids.data_ptr(), ts.data_ptr(), None if gs is None else gs.data_ptr(),
                                        self._freqs.data_ptr(), None if seqlens is None else seqlens.data_ptr(), st),
              "vcb_flux_prepare")
        self._shape = (B, Li, Lt, E)

    def forward(self, eval_idx: int, img: Tensor, out: Tensor | None = None) -> Tensor:
        """One Flux.forward with the tables of evaluation ``eval_idx``: img [B, Li, in_channels] -> [B, Li, out_channels]."""
        if self._shape is None:
            raise _lib.VcbError("FluxEngine.forward called before prepare")
        B, Li, Lt, E = self._shape
        if img.ndim != 3:
            raise ValueError("Input img and txt tensors must have 3 dimensions.")
        if tuple(img.shape) != (B, Li, self.params.in_channels):
            raise ValueError(f"img must be {(B, Li, self.params.in_channels)}, got {tuple(img.shape)}")
        if img.dtype != BF16 or not img.is_cuda or img.stride(2) != 1 or img.stride(0) != Li * img.stride(1):
            img = img.to(self.device, BF16).contiguous()
        if out is None:
            out = torch.empty(B, Li, self.params.out_channels, dtype=BF16, device=self.device)
        check(self.lib.vcb_flux_forward(self._h, eval_idx, img.data_ptr(), img.stride(1), out.data_ptr(), out.stride(1),
                                        torch.cuda.current_stream().cuda_stream), "vcb_flux_forward")
        return out
