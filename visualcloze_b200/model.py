"""FLUX-DiT container with the reference's call signature and state-dict contract, running on libvcb200.

Mirror of ``models/model.py`` (``FluxParams`` :18-32, ``Flux`` :35-151, ``FluxLoraWrapper`` :154-175):

  * ``Flux.forward(img, img_ids, txt, txt_ids, timesteps, y, txt_mask, img_mask, guidance)`` returns
    ``Tensor[B, Li, out_channels]`` in bf16, raises ``ValueError`` on non-3-D ``img``/``txt`` and on missing
    guidance exactly like the reference (:97-98, :104-105), never mutates its inputs;
  * ``state_dict()`` keys and shapes equal the reference's (``img_in.weight``,
    ``double_blocks.{i}.img_attn.qkv.lora_A.weight`` ...; SURVEY.md 8b "Weights"), so BFL safetensors and the
    LoRA checkpoint load with the reference's own ``load_state_dict(..., strict=False)`` sequence
    (``visualcloze.py:111-112``);
  * ``FluxLoraWrapper.set_lora_scale`` keeps its meaning.  By default LoRA is merged into packed weights
    (``W' = W + s * B A``, ``b' = b + s * b_B``), re-packed when the scale or a parameter changes: a second copy of
    the weights.  ``set_lora_mode("unmerged")`` runs it as the reference does, ``base(x) + s * B(A(x))``, on the
    module's own tensors: a scale change or an adapter swap (``load_state_dict(sd, strict=False, assign=True)``)
    then only rebuilds pointers and bias vectors, at about 8 % more GEMM work per evaluation.

The module holds parameters only; all arithmetic happens in the CUDA library (``engine.py``).  There is no
PyTorch fallback: calling ``forward`` without an H100 raises.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field

import torch
from torch import Tensor, nn

from .engine import FluxEngine, first_block_cache_threshold

BF16 = torch.bfloat16


@dataclass
class FluxParams:
    in_channels: int
    out_channels: int
    vec_in_dim: int
    context_in_dim: int
    hidden_size: int
    mlp_ratio: float
    num_heads: int
    depth: int
    depth_single_blocks: int
    axes_dim: list[int]
    theta: int
    qkv_bias: bool
    guidance_embed: bool


def flux_dev_fill_params() -> FluxParams:
    """``configs["flux-dev-fill-lora"].params`` (models/util.py:132-165): FLUX.1-Fill-dev geometry."""
    return FluxParams(in_channels=384, out_channels=64, vec_in_dim=768, context_in_dim=4096, hidden_size=3072,
                      mlp_ratio=4.0, num_heads=24, depth=19, depth_single_blocks=38, axes_dim=[16, 56, 56],
                      theta=10_000, qkv_bias=True, guidance_embed=True)


def linear_table(p: FluxParams) -> list[tuple[str, int, int]]:
    """(module path, in_features, out_features) for every nn.Linear of the reference model."""
    H, M = p.hidden_size, int(p.hidden_size * p.mlp_ratio)
    t = [("img_in", p.in_channels, H), ("time_in.in_layer", 256, H), ("time_in.out_layer", H, H),
         ("vector_in.in_layer", p.vec_in_dim, H), ("vector_in.out_layer", H, H)]
    if p.guidance_embed:
        t += [("guidance_in.in_layer", 256, H), ("guidance_in.out_layer", H, H)]
    t += [("txt_in", p.context_in_dim, H)]
    for i in range(p.depth):
        for s in ("img", "txt"):
            b = f"double_blocks.{i}.{s}"
            t += [(f"{b}_mod.lin", H, 6 * H), (f"{b}_attn.qkv", H, 3 * H), (f"{b}_attn.proj", H, H),
                  (f"{b}_mlp.0", H, M), (f"{b}_mlp.2", M, H)]
    for i in range(p.depth_single_blocks):
        b = f"single_blocks.{i}"
        t += [(f"{b}.linear1", H, 3 * H + M), (f"{b}.linear2", H + M, H), (f"{b}.modulation.lin", H, 3 * H)]
    t += [("final_layer.linear", H, p.out_channels), ("final_layer.adaLN_modulation.1", H, 2 * H)]
    return t


def norm_scale_names(p: FluxParams) -> list[str]:
    n = []
    for i in range(p.depth):
        for s in ("img", "txt"):
            n += [f"double_blocks.{i}.{s}_attn.norm.query_norm.scale", f"double_blocks.{i}.{s}_attn.norm.key_norm.scale"]
    for i in range(p.depth_single_blocks):
        n += [f"single_blocks.{i}.norm.query_norm.scale", f"single_blocks.{i}.norm.key_norm.scale"]
    return n


class _Node(nn.Module):
    """Anonymous container: the parameter tree is built from ``linear_table`` rather than from block classes."""


def _attach(root: nn.Module, dotted: str, param: nn.Parameter) -> None:
    parts = dotted.split(".")
    node = root
    for name in parts[:-1]:
        child = node._modules.get(name)
        if child is None:
            child = _Node()
            node.add_module(name, child)
        node = child
    node.register_parameter(parts[-1], param)


class Flux(nn.Module):
    """Transformer model for flow matching on sequences (reference: models/model.py:35-124)."""

    def __init__(self, params: FluxParams, device=None, dtype=BF16):
        super().__init__()
        self.params = params
        self.in_channels = params.in_channels
        self.out_channels = params.out_channels
        if params.hidden_size % params.num_heads != 0:
            raise ValueError(f"Hidden size {params.hidden_size} must be divisible by num_heads {params.num_heads}")
        pe_dim = params.hidden_size // params.num_heads
        if sum(params.axes_dim) != pe_dim:
            raise ValueError(f"Got {params.axes_dim} but expected positional dim {pe_dim}")
        if pe_dim != 128:
            raise ValueError("the sm_90a kernels are specialised for head_dim 128")
        self.hidden_size = params.hidden_size
        self.num_heads = params.num_heads
        self.lora_rank = 0
        self.lora_scale = 1.0
        self._engine: FluxEngine | None = None
        self._packed_key = None
        # names of the parameters that have received values (load_state_dict / init_synthetic / mark_initialized): base weights
        # are allocated with torch.empty, and packing an engine from never-loaded memory must fail loudly, not render garbage
        self._initialized: set[str] = set()
        self.linear_precision = "bf16"
        self.lora_mode = "merged"
        self._sp = None
        self._fbc = 0.0
        self._fbc_per_sample = False
        kw = dict(device=device, dtype=dtype)
        for name, fin, fout in linear_table(params):
            _attach(self, name + ".weight", nn.Parameter(torch.empty(fout, fin, **kw), requires_grad=False))
            if not (name.endswith("_attn.qkv") and not params.qkv_bias):
                _attach(self, name + ".bias", nn.Parameter(torch.empty(fout, **kw), requires_grad=False))
        for name in norm_scale_names(params):
            _attach(self, name, nn.Parameter(torch.ones(128, **kw), requires_grad=False))

    # ------------------------------------------------------------------------------------------
    def init_synthetic(self, seed: int = 0) -> "Flux":
        """Random weights of the right geometry, drawn on the parameters' device (benchmarks have no checkpoint):
        ``weight ~ N(0, 1/fan_in)`` with residual-branch output projections scaled by ``1/sqrt(n_blocks)``,
        ``bias, lora_B ~ N(0, 0.02^2)``, norm scales ``1 + N(0, 0.1^2)``."""
        nblk = max(1, self.params.depth + self.params.depth_single_blocks)
        dev = next(self.parameters()).device
        g = torch.Generator(device=dev).manual_seed(seed)
        with torch.no_grad():
            for name, p in self.named_parameters():
                if name.endswith(".scale"):
                    p.copy_(1.0 + 0.1 * torch.randn(p.shape, generator=g, device=dev))
                elif name.endswith("lora_B.weight") or name.endswith(".bias"):
                    p.copy_(0.02 * torch.randn(p.shape, generator=g, device=dev))
                else:
                    std = 1.0 / math.sqrt(p.shape[1])
                    if (".proj.weight" in name or "_mlp.2.weight" in name or "linear2.weight" in name) and "lora" not in name:
                        std /= math.sqrt(nblk)
                    p.copy_(std * torch.randn(p.shape, generator=g, device=dev))
        self._packed_key = None
        self._initialized = {n for n, _ in self.named_parameters()}
        return self

    def load_state_dict(self, state_dict, strict: bool = True, assign: bool = False):
        """``nn.Module.load_state_dict`` that also records which parameters received values (see ``uninitialized``)."""
        res = super().load_state_dict(state_dict, strict=strict, assign=assign)
        own = {n for n, _ in self.named_parameters()}
        self._initialized |= own & set(state_dict.keys())
        return res

    def mark_initialized(self, names=None) -> None:
        """Declare parameters filled by other means (``p.copy_`` ...) as initialised; ``None`` = all of them."""
        self._initialized |= {n for n, _ in self.named_parameters()} if names is None else set(names)

    def uninitialized(self) -> list[str]:
        """Base parameters still holding ``torch.empty`` memory.  QK-norm scales (ones) and the LoRA tensors (zero update)
        have well-defined defaults, exactly like the reference modules (layers.py:66, lora.py:84-86)."""
        return [n for n, _ in self.named_parameters()
                if n not in self._initialized and not n.endswith(".scale") and ".lora_" not in n]

    def engine(self) -> FluxEngine:
        """Packed-weight engine, rebuilt when a parameter was replaced or modified in place or the LoRA scale changed."""
        missing = self.uninitialized()
        if missing:
            from ._lib import VcbError
            raise VcbError(f"{len(missing)} base parameters were never loaded (e.g. {missing[:3]}): load the FLUX.1-Fill checkpoint "
                           "(VisualClozeModel(flux_ckpt=...) / load_state_dict) or call init_synthetic() before running the model")
        key = (self.lora_scale, self.linear_precision, self.lora_mode) + tuple((p.data_ptr(), p._version) for p in self.parameters())
        if self._engine is None or key != self._packed_key:
            ws = self._engine._ws if self._engine is not None else None     # the device workspace carries over
            self._engine = None                     # release the previous packing before building the next one
            self._engine = FluxEngine(self.params, dict(self.named_parameters()), self.lora_scale,
                                      fp8={"bf16": 0, "fp8": 1, "fp8_all": 2}[self.linear_precision], lora_mode=self.lora_mode,
                                      workspace=ws)
            self._packed_key = key
            if getattr(self, "_sp", None) is not None:
                self._engine.enable_sequence_parallel(self._sp)
            if self._fbc:
                self._engine.set_first_block_cache(self._fbc, self._fbc_per_sample)
        return self._engine

    def set_linear_precision(self, precision: str) -> None:
        """"bf16" (default; the reference's numerics) or "fp8": the LayerNorm-fed projections (qkv, mlp.0, linear1 -- 58 % of the
        step's GEMM FLOPs) run on e4m3 operands with per-row activation / per-channel weight scales.  Opt-in, NOT the reference's
        numerics: see DESIGN.md (fp8 contract) for the measured deviation.  "fp8_all" adds the gated-residual Linears (attn.proj,
        mlp.2, linear2: every GEMM of the blocks), whose bf16 inputs are quantised row-wise first -- faster, and further from the
        bf16 path (its own numbers in the same contract).  No counterpart in the reference."""
        if precision not in ("bf16", "fp8", "fp8_all"):
            raise ValueError("linear precision must be 'bf16', 'fp8' or 'fp8_all'")
        if precision != "bf16" and self.lora_mode == "unmerged":
            raise ValueError("the fp8 projections need merged LoRA weights (set_lora_mode('merged') first)")
        self.linear_precision = precision

    def set_lora_mode(self, mode: str) -> None:
        """"merged" (default): the engine packs ``W + s * B A`` once, a second copy of every weight, and re-merges when the scale
        or a parameter changes.  "unmerged": every call computes ``base(x) + s * B(A(x))`` like the reference's LinearLora
        (lora.py:92-98), on the module's own tensors; changing the scale or swapping adapters costs a bias rebuild, each
        evaluation about 8 % more GEMM work.  Which is better depends on how often the adapter or scale changes and on how
        much memory other resident models need.  Unmerged takes bf16 projections on one GPU: it refuses fp8 precisions and
        sequence parallelism."""
        if mode not in ("merged", "unmerged"):
            raise ValueError("lora mode must be 'merged' or 'unmerged'")
        if mode == "unmerged":
            if self.linear_precision != "bf16":
                raise ValueError("unmerged LoRA runs on bf16 operands (set_linear_precision('bf16') first)")
            if self._sp is not None and self._sp.world > 1:
                raise ValueError("sequence-parallel mode takes merged LoRA weights only")
        self.lora_mode = mode

    def enable_sequence_parallel(self, sp) -> None:
        """Single-image latency mode over several GPUs (``parallel.SequenceParallel``; None switches it off).  No counterpart
        in the reference (single-GPU inference); the call signature and the results' contract are unchanged: every rank
        passes the same full inputs and receives the same full output.  Needs merged LoRA weights."""
        if sp is not None and sp.world > 1 and self.lora_mode == "unmerged":
            raise ValueError("sequence-parallel mode takes merged LoRA weights only (set_lora_mode('merged') first)")
        if sp is not None and sp.world > 1 and self._fbc:
            raise ValueError("the first-block cache decides per batch on one GPU (enable_first_block_cache(None) first)")
        self._sp = sp
        if self._engine is not None:
            self._engine.enable_sequence_parallel(sp)

    def enable_first_block_cache(self, threshold: float | None, per_sample: bool = False) -> None:
        """Opt-in first-block cache (FBCache; no counterpart in the reference, NOT the reference's numerics).  Within one sampler
        solve, every evaluation runs double block 0; when its img-row residual differs from the one of the last fully computed
        evaluation by less than ``threshold`` (sum|r - r_ref| / sum|r_ref| over the valid rows of the whole batch), the other blocks
        are skipped and their residual from that evaluation is reused.  The first evaluation of a solve is always computed.
        ``None`` or 0 switches it off (the default).  Composes with both LoRA modes and the fp8 precisions; refused with sequence
        parallelism.  No threshold is recommended: quality on trained weights has not been measured (DESIGN.md §2d).
        ``per_sample``: decide every sample of a batch on its own rows (DESIGN.md §2g), so that a request's output does not depend
        on the other requests it shares a batched solve with; at batch 1 both modes give the same bits."""
        t = first_block_cache_threshold(threshold)
        if not isinstance(per_sample, bool):
            raise ValueError(f"per_sample must be a bool, got {per_sample!r}")
        if t > 0 and self._sp is not None and self._sp.world > 1:
            raise ValueError("the first-block cache decides per batch on one GPU; it is refused with sequence parallelism")
        self._fbc, self._fbc_per_sample = t, per_sample
        if self._engine is not None:
            self._engine.set_first_block_cache(t, per_sample)

    def cache_stats(self, per_sample: bool = False):
        """First-block cache counters of the latest solve (or ``forward``): evaluations "computed" and "skipped" and the latest
        "last_diff" (inf for the first evaluation of a solve, NaN before any).  In per-sample mode an evaluation counts as skipped
        when every sample skipped, and "last_diff" is the largest sample's.  ``per_sample=True``: a list with those counters for
        each sample of the latest solve (each sample's own in per-sample mode, the batch's otherwise)."""
        if per_sample:
            if self._engine is None or self._engine._shape is None:
                return []
            return self._engine.sample_cache_stats()
        if self._engine is None:
            return {"computed": 0, "skipped": 0, "last_diff": math.nan}
        return self._engine.cache_stats()

    # ------------------------------------------------------------------------------------------
    def forward(self, img: Tensor, img_ids: Tensor, txt: Tensor, txt_ids: Tensor, timesteps: Tensor, y: Tensor,
                txt_mask: Tensor = None, img_mask: Tensor = None, guidance: Tensor | None = None) -> Tensor:
        if img.ndim != 3 or txt.ndim != 3:
            raise ValueError("Input img and txt tensors must have 3 dimensions.")
        if self.params.guidance_embed and guidance is None:
            raise ValueError("Didn't get guidance strength for guidance distilled model.")
        eng = self.engine()
        eng.prepare(txt=txt, y=y, img_ids=img_ids, txt_ids=txt_ids, timesteps=timesteps[None], guidance=guidance,
                    txt_mask=txt_mask, img_mask=img_mask, n_img_tokens=img.shape[1])
        if eng._sp is not None:        # sequence-parallel: every rank passes the full inputs and gets the full output
            out = eng._sp.gather(eng.forward(0, eng._sp.shard(img)), dim=1)
            eng._sp.check()
            return out
        return eng.forward(0, img)

    def get_fsdp_wrap_module_list(self):      # training-side helpers of the reference; inference-only here
        return []

    def get_checkpointing_wrap_module_list(self):
        return []


class FluxLoraWrapper(Flux):
    """models/model.py:154-175: every Linear gets ``lora_A [r, in]``, ``lora_B [out, r]`` (+ bias), r = min(rank, in, out)."""

    def __init__(self, lora_rank: int = 128, lora_scale: float = 1.0, *args, **kwargs) -> None:
        super().__init__(*args, **kwargs)
        self.lora_rank = lora_rank
        self.lora_scale = float(lora_scale)
        some = next(self.parameters())
        kw = dict(device=some.device, dtype=some.dtype)
        for name, fin, fout in linear_table(self.params):
            r = min(lora_rank, fin, fout)
            # zero default (the reference draws lora_A at random, lora.py:84; with lora_B = 0 the update is zero either way, and
            # zeros cannot inject NaNs from uninitialised memory into the merged weight)
            _attach(self, name + ".lora_A.weight", nn.Parameter(torch.zeros(r, fin, **kw), requires_grad=False))
            # the reference zero-initialises lora_B (lora.py:84-86)
            _attach(self, name + ".lora_B.weight", nn.Parameter(torch.zeros(fout, r, **kw), requires_grad=False))
            _attach(self, name + ".lora_B.bias", nn.Parameter(torch.zeros(fout, **kw), requires_grad=False))

    def set_lora_scale(self, scale: float) -> None:
        assert isinstance(scale, float), "scalar value must be a float"
        self.lora_scale = scale
