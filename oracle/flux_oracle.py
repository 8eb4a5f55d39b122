"""CPU oracle for the VisualCloze FLUX-DiT forward -- TEST INFRASTRUCTURE ONLY.

This file is a checker, not a product path.  Only ``tests/``, ``__graft_entry__.smoke()``
and the ``cpu_baseline`` / ``--impl reference`` legs of ``bench.py`` may import it.  The
shipped path (``visualcloze_b200``) never imports anything from ``oracle/``.

It restates, as flat functions over a reference-named state dict, the algorithm of

  * ``models/model.py:85-124``            (Flux.forward)
  * ``models/modules/layers.py:11-259``   (EmbedND, timestep_embedding, MLPEmbedder, RMSNorm,
                                            QKNorm, Modulation, Double/SingleStreamBlock, LastLayer)
  * ``models/math.py:63-117``             (attention, rope, apply_rope)
  * ``models/modules/lora.py:92-98``      (LinearLora.forward, un-merged)

with the dtype behaviour the reference gets from ``torch.autocast`` written out as explicit
casts.  Three numerics modes:

  ``cuda_bf16``  what the reference does under ``torch.autocast("cuda", bf16)``
                 (``visualcloze.py:363``): Linear in bf16, LayerNorm returns fp32, modulate in
                 fp32, RMSNorm/RoPE fp32 math with bf16 results, bf16 residual stream.  This is
                 the mode the CUDA kernels are checked against.
  ``cpu_bf16``   the same under ``torch.autocast("cpu", bf16)``: identical except LayerNorm is
                 not on the CPU autocast fp32 list, so it returns bf16.  Used to pin this file
                 against the reference modules executed in the build container
                 (``oracle/gen_golden.py`` -> ``tests/golden/``).
  ``fp32``       everything fp32; pins structure/conventions against the fp32 reference.

Pinning status: the reference has no tests or golden vectors (SURVEY.md section 4), so this
oracle is pinned against outputs of the reference modules themselves, generated in the build
container by ``oracle/gen_golden.py`` and committed under ``tests/golden/``.
"""
from __future__ import annotations

import collections.abc
import math
from dataclasses import dataclass, field

import torch
import torch.nn.functional as F

BF16 = torch.bfloat16
F32 = torch.float32


@dataclass
class FluxConfig:
    """Mirror of ``FluxParams`` (models/model.py:18-32) + LoRA wrapper args (:154-170)."""

    in_channels: int = 384
    out_channels: int = 64
    vec_in_dim: int = 768
    context_in_dim: int = 4096
    hidden_size: int = 3072
    mlp_ratio: float = 4.0
    num_heads: int = 24
    depth: int = 19
    depth_single_blocks: int = 38
    axes_dim: list = field(default_factory=lambda: [16, 56, 56])
    theta: int = 10_000
    qkv_bias: bool = True
    guidance_embed: bool = True
    lora_rank: int = 256
    lora_scale: float = 1.0

    @property
    def head_dim(self) -> int:
        return self.hidden_size // self.num_heads

    @property
    def mlp_hidden(self) -> int:
        return int(self.hidden_size * self.mlp_ratio)


class Numerics:
    def __init__(self, mode: str = "cuda_bf16"):
        assert mode in ("cuda_bf16", "cpu_bf16", "fp32")
        self.mode = mode
        self.cd = F32 if mode == "fp32" else BF16          # autocast "lower precision" dtype
        self.ln_dtype = BF16 if mode == "cpu_bf16" else F32  # dtype LayerNorm returns


# ----------------------------------------------------------------------------------------------
# parameter shapes (state-dict contract, SURVEY.md 8b "Weights")
# ----------------------------------------------------------------------------------------------
def linear_names(cfg: FluxConfig) -> list[tuple[str, int, int]]:
    """(module path, in_features, out_features) of every nn.Linear in Flux, reference order."""
    H, M = cfg.hidden_size, cfg.mlp_hidden
    out = [("img_in", cfg.in_channels, H),
           ("time_in.in_layer", 256, H), ("time_in.out_layer", H, H),
           ("vector_in.in_layer", cfg.vec_in_dim, H), ("vector_in.out_layer", H, H)]
    if cfg.guidance_embed:
        out += [("guidance_in.in_layer", 256, H), ("guidance_in.out_layer", H, H)]
    out += [("txt_in", cfg.context_in_dim, H)]
    for i in range(cfg.depth):
        p = f"double_blocks.{i}."
        for s in ("img", "txt"):
            out += [(p + f"{s}_mod.lin", H, 6 * H), (p + f"{s}_attn.qkv", H, 3 * H),
                    (p + f"{s}_attn.proj", H, H), (p + f"{s}_mlp.0", H, M), (p + f"{s}_mlp.2", M, H)]
    for i in range(cfg.depth_single_blocks):
        p = f"single_blocks.{i}."
        out += [(p + "linear1", H, 3 * H + M), (p + "linear2", H + M, H), (p + "modulation.lin", H, 3 * H)]
    out += [("final_layer.linear", H, cfg.out_channels), ("final_layer.adaLN_modulation.1", H, 2 * H)]
    return out


def param_shapes(cfg: FluxConfig, lora: bool = True) -> dict[str, tuple]:
    """name -> shape for the full state dict (base + LoRA), matching FluxLoraWrapper.state_dict()."""
    shapes: dict[str, tuple] = {}
    for name, fin, fout in linear_names(cfg):
        shapes[name + ".weight"] = (fout, fin)
        if name.endswith("_attn.qkv") and not cfg.qkv_bias:
            pass
        else:
            shapes[name + ".bias"] = (fout,)
        if lora and cfg.lora_rank > 0:
            r = min(cfg.lora_rank, fin, fout)           # lora.py:67-68
            shapes[name + ".lora_A.weight"] = (r, fin)
            shapes[name + ".lora_B.weight"] = (fout, r)
            shapes[name + ".lora_B.bias"] = (fout,)
    D = cfg.head_dim
    for i in range(cfg.depth):
        for s in ("img", "txt"):
            shapes[f"double_blocks.{i}.{s}_attn.norm.query_norm.scale"] = (D,)
            shapes[f"double_blocks.{i}.{s}_attn.norm.key_norm.scale"] = (D,)
    for i in range(cfg.depth_single_blocks):
        shapes[f"single_blocks.{i}.norm.query_norm.scale"] = (D,)
        shapes[f"single_blocks.{i}.norm.key_norm.scale"] = (D,)
    return shapes


def make_params(cfg: FluxConfig, seed: int = 0, lora: bool = True, dtype=BF16,
                w_std: float | None = None) -> dict[str, torch.Tensor]:
    """Deterministic synthetic weights, independent of module construction order.

    Parameters are drawn in sorted-name order from one CPU generator:
    ``weight ~ N(0, 1/fan_in)`` (so activations stay O(1)), ``bias ~ N(0, 0.02^2)``,
    ``lora_A ~ N(0, 1/fan_in)``, ``lora_B ~ N(0, 0.02^2)`` (re-randomised: the reference's zero
    init would hide the LoRA branch, lora.py:84-86), RMSNorm scales ``1 + N(0, 0.1^2)``.
    Residual-branch output projections are additionally scaled by ``1/sqrt(n_blocks)`` to keep
    the 57-block residual stream bounded in bf16.
    """
    g = torch.Generator().manual_seed(seed)
    shapes = param_shapes(cfg, lora)
    nblk = max(1, cfg.depth + cfg.depth_single_blocks)
    out = {}
    for name in sorted(shapes):
        shp = shapes[name]
        if name.endswith(".scale"):
            t = 1.0 + 0.1 * torch.randn(shp, generator=g)
        elif name.endswith("lora_B.weight") or name.endswith(".bias"):
            t = 0.02 * torch.randn(shp, generator=g)
        else:
            std = w_std if w_std is not None else 1.0 / math.sqrt(shp[1])
            t = std * torch.randn(shp, generator=g)
            if (".proj.weight" in name or "_mlp.2.weight" in name or "linear2.weight" in name) \
                    and "lora" not in name:
                t = t / math.sqrt(nblk)
        out[name] = t.to(dtype)
    return out


# ----------------------------------------------------------------------------------------------
# building blocks
# ----------------------------------------------------------------------------------------------
def lora_linear(p: dict, name: str, x: torch.Tensor, nm: Numerics, scale: float) -> torch.Tensor:
    """LinearLora.forward (lora.py:92-98) under autocast: three bf16 Linears, bf16 mul and add."""
    cd = nm.cd
    w = p[name + ".weight"].to(cd)
    b = p.get(name + ".bias")
    y = F.linear(x.to(cd), w, None if b is None else b.to(cd))
    a = p.get(name + ".lora_A.weight")
    if a is not None:
        t = F.linear(x.to(cd), a.to(cd))
        bb = p.get(name + ".lora_B.bias")
        u = F.linear(t, p[name + ".lora_B.weight"].to(cd), None if bb is None else bb.to(cd))
        y = y + u * scale
    return y


def timestep_embedding(t: torch.Tensor, dim: int = 256, max_period: int = 10000,
                       time_factor: float = 1000.0) -> torch.Tensor:
    """layers.py:28-49.  Result has t's dtype (fp32 timesteps, bf16 guidance)."""
    t = time_factor * t
    half = dim // 2
    freqs = torch.exp(-math.log(max_period) * torch.arange(0, half, dtype=F32) / half).to(t.device)
    args = t[:, None].float() * freqs[None]
    emb = torch.cat([torch.cos(args), torch.sin(args)], dim=-1)
    return emb.to(t.dtype) if torch.is_floating_point(t) else emb


def mlp_embedder(p, name, x, nm, ls):
    """layers.py:52-60."""
    return lora_linear(p, name + ".out_layer", F.silu(lora_linear(p, name + ".in_layer", x, nm, ls)), nm, ls)


def rope_table(ids: torch.Tensor, axes_dim, theta: int) -> tuple[torch.Tensor, torch.Tensor]:
    """EmbedND + rope (layers.py:11-25, math.py:102-109) as (cos, sin) of shape [B, L, D/2] fp32.

    The reference stores 2x2 matrices [[cos, -sin], [sin, cos]]; cos/sin carry the same numbers.
    """
    cs, sn = [], []
    for i, d in enumerate(axes_dim):
        scale = torch.arange(0, d, 2, dtype=torch.float64, device=ids.device) / d
        omega = 1.0 / (theta ** scale)
        ang = ids[..., i].double()[..., None] * omega
        cs.append(torch.cos(ang).float())
        sn.append(torch.sin(ang).float())
    return torch.cat(cs, -1), torch.cat(sn, -1)


def apply_rope(x: torch.Tensor, cos: torch.Tensor, sin: torch.Tensor) -> torch.Tensor:
    """math.py:112-117 for one tensor x [B, H, L, D]; fp32 math, result in x.dtype."""
    xf = x.float().reshape(*x.shape[:-1], -1, 2)
    x0, x1 = xf[..., 0], xf[..., 1]
    c, s = cos[:, None], sin[:, None]
    o0 = c * x0 + (-s) * x1
    o1 = s * x0 + c * x1
    return torch.stack([o0, o1], -1).reshape(x.shape).to(x.dtype)


def rms_norm(x: torch.Tensor, scale: torch.Tensor) -> torch.Tensor:
    """RMSNorm.forward (layers.py:68-72): fp32 stats, cast back, then multiply by the scale."""
    xd = x.dtype
    xf = x.float()
    rrms = torch.rsqrt(torch.mean(xf * xf, dim=-1, keepdim=True) + 1e-6)
    return (xf * rrms).to(xd) * scale.to(xd)


def joint_attention(q, k, v, cos, sin, mask, nm: Numerics) -> torch.Tensor:
    """attention() (math.py:63-99): RoPE, softmax(QK^T/sqrt(D))V over keys with mask==1,
    padded query rows zeroed (pad_input).  q,k,v [B,H,L,D] -> [B, L, H*D].

    Mirrors flash-attn numerics: fp32 scores/softmax, probabilities rounded to the compute
    dtype before the PV product, fp32 accumulation, row-sum taken from the unrounded fp32 P.
    """
    q = apply_rope(q, cos, sin)
    k = apply_rope(k, cos, sin)
    B, H, L, D = q.shape
    s = torch.matmul(q.float(), k.float().transpose(-1, -2)) * (D ** -0.5)
    if mask is not None:
        s = s.masked_fill(mask[:, None, None, :] == 0, float("-inf"))
    m = s.amax(-1, keepdim=True)
    pexp = torch.exp(s - m)
    den = pexp.sum(-1, keepdim=True)
    o = torch.matmul(pexp.to(nm.cd).float(), v.float()) / den
    o = o.to(nm.cd)
    if mask is not None:
        o = o * mask[:, None, :, None].to(o.dtype)
    return o.permute(0, 2, 1, 3).reshape(B, L, H * D)


def _split_heads(x: torch.Tensor, H: int):
    """"B L (K H D) -> K B H L D" (layers.py:166)."""
    B, L, _ = x.shape
    x = x.reshape(B, L, 3, H, -1).permute(2, 0, 3, 1, 4)
    return x[0], x[1], x[2]


def _modulate(x: torch.Tensor, shift, scale, nm: Numerics) -> torch.Tensor:
    """(1 + scale) * LayerNorm(x) + shift  (layers.py:163-164).  `1 + scale` is a bf16 op."""
    ln = F.layer_norm(x.to(nm.ln_dtype), (x.shape[-1],), eps=1e-6)
    return (1 + scale) * ln + shift


def modulation(p, name, vec, nm, ls, n):
    """Modulation.forward (layers.py:120-126): n chunks of [B,1,H]."""
    return lora_linear(p, name, F.silu(vec), nm, ls)[:, None, :].chunk(n, dim=-1)


def double_block(p, i, cfg, img, txt, vec, cos, sin, mask, nm, ls):
    """DoubleStreamBlock.forward (layers.py:158-196)."""
    pre = f"double_blocks.{i}."
    H = cfg.num_heads
    Lt = txt.shape[1]
    qs, ks, vs, mods = {}, {}, {}, {}
    for s, x in (("txt", txt), ("img", img)):
        m = modulation(p, pre + f"{s}_mod.lin", vec, nm, ls, 6)
        mods[s] = m
        xm = _modulate(x, m[0], m[1], nm)
        q, k, v = _split_heads(lora_linear(p, pre + f"{s}_attn.qkv", xm, nm, ls), H)
        qs[s] = rms_norm(q, p[pre + f"{s}_attn.norm.query_norm.scale"]).to(v.dtype)
        ks[s] = rms_norm(k, p[pre + f"{s}_attn.norm.key_norm.scale"]).to(v.dtype)
        vs[s] = v
    q = torch.cat((qs["txt"], qs["img"]), 2)
    k = torch.cat((ks["txt"], ks["img"]), 2)
    v = torch.cat((vs["txt"], vs["img"]), 2)
    attn = joint_attention(q, k, v, cos, sin, mask, nm)
    outs = {}
    for s, x, a in (("img", img, attn[:, Lt:]), ("txt", txt, attn[:, :Lt])):
        m = mods[s]
        x = x + m[2] * lora_linear(p, pre + f"{s}_attn.proj", a, nm, ls)
        h = _modulate(x, m[3], m[4], nm)
        h = lora_linear(p, pre + f"{s}_mlp.0", h, nm, ls)
        h = F.gelu(h, approximate="tanh")
        h = lora_linear(p, pre + f"{s}_mlp.2", h, nm, ls)
        outs[s] = x + m[5] * h
    return outs["img"], outs["txt"]


def single_block(p, i, cfg, x, vec, cos, sin, mask, nm, ls):
    """SingleStreamBlock.forward (layers.py:232-245)."""
    pre = f"single_blocks.{i}."
    Hd = cfg.hidden_size
    shift, scale, gate = modulation(p, pre + "modulation.lin", vec, nm, ls, 3)
    xm = _modulate(x, shift, scale, nm)
    y = lora_linear(p, pre + "linear1", xm, nm, ls)
    qkv, mlp = y[..., : 3 * Hd], y[..., 3 * Hd:]
    q, k, v = _split_heads(qkv, cfg.num_heads)
    q = rms_norm(q, p[pre + "norm.query_norm.scale"]).to(v.dtype)
    k = rms_norm(k, p[pre + "norm.key_norm.scale"]).to(v.dtype)
    attn = joint_attention(q, k, v, cos, sin, mask, nm)
    out = lora_linear(p, pre + "linear2", torch.cat((attn, F.gelu(mlp, approximate="tanh")), 2), nm, ls)
    return x + gate * out


def last_layer(p, x, vec, nm, ls):
    """LastLayer.forward (layers.py:255-259); chunk order is (shift, scale)."""
    shift, scale = lora_linear(p, "final_layer.adaLN_modulation.1", F.silu(vec), nm, ls).chunk(2, dim=1)
    x = _modulate(x, shift[:, None, :], scale[:, None, :], nm)
    return lora_linear(p, "final_layer.linear", x, nm, ls)


def flux_vec(p, cfg, timesteps, y, guidance, nm, ls):
    """vec = time_in(temb(t)) + guidance_in(temb(g)) + vector_in(y)  (model.py:102-107)."""
    vec = mlp_embedder(p, "time_in", timestep_embedding(timesteps, 256), nm, ls)
    if cfg.guidance_embed:
        if guidance is None:
            raise ValueError("Didn't get guidance strength for guidance distilled model.")
        vec = vec + mlp_embedder(p, "guidance_in", timestep_embedding(guidance, 256), nm, ls)
    return vec + mlp_embedder(p, "vector_in", y, nm, ls)


class _Fp32View(collections.abc.Mapping):
    """The parameters in fp32, converted as they are read (a full-size model does not fit a device twice over)."""

    def __init__(self, p):
        self.p = p

    def __iter__(self):
        return iter(self.p)

    def __len__(self):
        return len(self.p)

    def __getitem__(self, k):
        return self.p[k].float()


def flux_forward(p: dict, cfg: FluxConfig, img, img_ids, txt, txt_ids, timesteps, y,
                 txt_mask=None, img_mask=None, guidance=None, mode: str = "cuda_bf16",
                 taps: dict | None = None) -> torch.Tensor:
    """Flux.forward (models/model.py:85-124).  ``taps`` (optional dict) receives intermediates."""
    if img.ndim != 3 or txt.ndim != 3:
        raise ValueError("Input img and txt tensors must have 3 dimensions.")
    nm = Numerics(mode)
    ls = cfg.lora_scale
    if mode == "fp32":
        p = _Fp32View(p)
        img, txt, y = img.float(), txt.float(), y.float()
        guidance = None if guidance is None else guidance.float()
    img = lora_linear(p, "img_in", img, nm, ls)
    vec = flux_vec(p, cfg, timesteps, y, guidance, nm, ls)
    txt = lora_linear(p, "txt_in", txt, nm, ls)
    ids = torch.cat((txt_ids, img_ids), dim=1)
    cos, sin = rope_table(ids, cfg.axes_dim, cfg.theta)
    mask = torch.cat((txt_mask, img_mask), dim=1)
    if taps is not None:
        taps.update(vec=vec, img_in=img, txt_in=txt, cos=cos, sin=sin)
    for i in range(cfg.depth):
        img, txt = double_block(p, i, cfg, img, txt, vec, cos, sin, mask, nm, ls)
        if taps is not None:
            taps[f"double.{i}.img"], taps[f"double.{i}.txt"] = img, txt
    x = torch.cat((txt, img), 1)
    for i in range(cfg.depth_single_blocks):
        x = single_block(p, i, cfg, x, vec, cos, sin, mask, nm, ls)
        if taps is not None:
            taps[f"single.{i}"] = x
    x = x[:, txt.shape[1]:, ...]
    return last_layer(p, x, vec, nm, ls)
