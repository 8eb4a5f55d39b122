"""``VisualClozeModel`` -- the reference's inference entry point on the H100-native hot path.

Mirror of ``visualcloze.py:78-467``: same constructor arguments, ``set_grid_size``, ``process_images`` and ``upsampling``
signatures and return types (list of PIL images / PIL image), same image preparation, mask/cond packing, seeding,
row-wise RoPE ids, sampler settings and output cropping.  What differs is where the work runs:

  * the flow model is ``visualcloze_b200.model.FluxLoraWrapper`` (libvcb200 kernels), driven through
    ``visualcloze_b200.transport.Sampler`` -- one ``vcb_flux_forward`` + one ``vcb_euler_update`` per step;
  * only the query (last) row is decoded, fused with un-patchify, scale/shift, ``(x + 1) / 2``, clamp and uint8
    conversion (the reference decodes every row and returns crops of the last one, visualcloze.py:424-453);
  * text encoders (T5-XXL / CLIP-L) are outside this path (SURVEY.md 2 #10, 8f): they are injected as callables --
    ``t5(list[str]) -> [B, 512, 4096]``, ``clip(list[str]) -> [B, 768]`` -- e.g. the reference's own ``load_t5`` /
    ``load_clip``;
  * the VAE *encode* of the condition rows (visualcloze.py:377-388) runs on ``vae.AutoEncoderEncoder`` (libvcb200; the
    "next" row (f)-1 of SURVEY.md section 8) unless an external ``encode(image [1, 3, H, W]) -> latent [1, 16, H/8, W/8]``
    callable (sampled, un-scaled -- e.g. ``AutoencoderKL.encode(...).latent_dist.sample()``) is injected.
"""
from __future__ import annotations

import random
from typing import NamedTuple

import numpy as np
import torch
from PIL import Image

from . import _lib as _vcb_lib, ops, resample
from .model import FluxLoraWrapper, flux_dev_fill_params
from .sampling import prepare_modified
from .transport import Sampler, create_transport
from .vae import AutoEncoderDecoder, AutoEncoderEncoder

_CONTENT_PREFIXES = (
    "The content of the last image in the final row is: ", "The last image of the last row depicts: ",
    "In the final row, the last image shows: ", "The last image in the bottom row illustrates: ",
    "The content of the bottom-right image is: ", "The final image in the last row portrays: ",
    "The last image of the final row displays: ", "In the last row, the final image captures: ",
    "The bottom-right corner image presents: ", "The content of the last image in the concluding row is: ",
    "In the last row, ", "The editing instruction in the last row is: ",
)


def aspect_ratio_size(size, resolution: int, divisible: int = 16, aspect_ratio=None) -> tuple:
    """The size ``resize_with_aspect_ratio`` resizes an image of ``size`` = (w, h) to."""
    w, h = size
    if aspect_ratio is None:
        aspect_ratio = w / h
    new_h = int((resolution * resolution / aspect_ratio) ** 0.5)
    new_w = int(new_h * aspect_ratio)
    new_w = max(new_w // divisible, 1) * divisible
    new_h = max(new_h // divisible, 1) * divisible
    return new_w, new_h


def resize_with_aspect_ratio(img: Image.Image, resolution: int, divisible: int = 16, aspect_ratio=None) -> Image.Image:
    """area ~= resolution^2, aspect kept, both sides multiples of 16 (visualcloze.py:28-75, PIL branch)."""
    return img.resize(aspect_ratio_size(img.size, resolution, divisible, aspect_ratio), Image.LANCZOS)


def to_rgb_if_rgba(img: Image.Image) -> Image.Image:
    """util/imgproc.py:90-96: composite RGBA over white."""
    if img.mode.upper() == "RGBA":
        rgb = Image.new("RGB", img.size, (255, 255, 255))
        rgb.paste(img, mask=img.split()[3])
        return rgb
    return img


def image_transform(img: Image.Image) -> torch.Tensor:
    """ToTensor + Normalize(0.5, 0.5): uint8 HWC -> float CHW in [-1, 1] (visualcloze.py:133-137)."""
    a = np.asarray(to_rgb_if_rgba(img).convert("RGB"), dtype=np.uint8)
    t = torch.from_numpy(a.copy()).permute(2, 0, 1).float().div(255.0)
    return (t - 0.5) / 0.5


def _pack_mask(mask: torch.Tensor) -> torch.Tensor:
    """[1,1,H,W] -> "b c (h 8)(w 8) -> b (c 8 8) h w" -> "b c (h 2)(w 2) -> b (h w) (c 2 2)" (visualcloze.py:381-382)."""
    b, c, H, W = mask.shape
    m = mask.reshape(b, c, H // 8, 8, W // 8, 8).permute(0, 1, 3, 5, 2, 4).reshape(b, c * 64, H // 8, W // 8)
    h, w = H // 16, W // 16
    return m.reshape(b, c * 64, h, 2, w, 2).permute(0, 2, 4, 1, 3, 5).reshape(b, h * w, c * 256)


def _patchify(lat: torch.Tensor) -> torch.Tensor:
    """"b c (h ph)(w pw) -> b (h w)(c ph pw)", ph = pw = 2."""
    b, c, H, W = lat.shape
    return lat.reshape(b, c, H // 2, 2, W // 2, 2).permute(0, 2, 4, 1, 3, 5).reshape(b, (H // 2) * (W // 2), c * 4)


class CellPlan(NamedTuple):
    """How one grid cell is made: start from the caller's image (``blank`` None) or from a black RGB image of size ``blank``
    (a missing target), then apply ``ops`` in order: ("resize", (w, h), filter) with filter ``resample.LANCZOS`` /
    ``resample.BICUBIC``, or ("crop", (left, top, right, bottom)) with Pillow's zero padding outside the image."""
    blank: tuple | None
    ops: tuple

    @property
    def size(self) -> tuple:
        """(w, h) of the finished cell"""
        if not self.ops:
            return self.blank
        op = self.ops[-1]
        return op[1] if op[0] == "resize" else (op[1][2] - op[1][0], op[1][3] - op[1][1])


def grid_plan(sizes, grid_h: int, grid_w: int, resolution: int):
    """The decisions of visualcloze.py:300-360 as a pure function of the input sizes, with the reference's quirks (the
    multi-target loop reassigns ``new_w``).  sizes[i][j]: (w, h) of cell (i, j), or None for a missing target of the last row.
    -> (cells: CellPlan per cell, row-major; mask_position; upsampling_size)."""
    cells, mask_position = [], []
    target_size = upsampling_size = None
    for i in range(grid_h):
        reference_size = None
        for j in range(grid_w):
            if sizes[i][j] is not None:
                if i == grid_h - 1 and upsampling_size is None:
                    upsampling_size = tuple(sizes[i][j])
                reference_size = aspect_ratio_size(sizes[i][j], resolution)
                if i == grid_h - 1 and target_size is None:
                    target_size = reference_size
                break
        for j in range(grid_w):
            if sizes[i][j] is not None:
                tw, th = aspect_ratio_size(sizes[i][j], resolution)
                if tw <= th:
                    size = (reference_size[0], int(reference_size[0] / tw * th))
                else:
                    size = (int(reference_size[1] / th * tw), reference_size[1])
                left, top = (size[0] - reference_size[0]) // 2, (size[1] - reference_size[1]) // 2      # center_crop
                cells.append(CellPlan(None, (("resize", (tw, th), resample.LANCZOS), ("resize", size, resample.BICUBIC),
                                             ("crop", (left, top, left + reference_size[0], top + reference_size[1])))))
                if i == grid_h - 1:
                    mask_position.append(0)
            else:
                if i != grid_h - 1:
                    raise ValueError("Please provide each image in the in-context example.")
                cells.append(CellPlan(reference_size or (resolution, resolution), ()))
                mask_position.append(1)
    if len(mask_position) > 1 and sum(mask_position) > 1:
        new_w = 384 if target_size is None else target_size[0]
        for k, cell in enumerate(cells):
            w, h = cell.size
            new_h = int(h * (new_w / w))
            new_w, new_h = int(new_w / 16) * 16, int(new_h / 16) * 16
            cells[k] = cell._replace(ops=cell.ops + (("resize", (new_w, new_h), resample.BICUBIC),))
    return cells, mask_position, upsampling_size


_PIL_FILTERS = {resample.LANCZOS: Image.LANCZOS, resample.BICUBIC: Image.BICUBIC}


def run_cell_pil(image, cell: CellPlan) -> Image.Image:
    """One CellPlan executed with Pillow."""
    im = image if cell.blank is None else Image.new("RGB", cell.blank, (0, 0, 0))
    for op in cell.ops:
        im = im.resize(op[1], _PIL_FILTERS[op[2]]) if op[0] == "resize" else im.crop(op[1])
    return im


def run_cell_device(image: torch.Tensor | None, cell: CellPlan, out: torch.Tensor, col0: int) -> None:
    """One CellPlan executed on the device: image uint8 [h, w, 3] CUDA (None for a blank cell) -> ``image_transform`` of the
    cell into out[:, :, col0:col0 + w] (out fp32 [3, h, W]).  A crop that ends the plan is done by the store."""
    im, ops_ = image, cell.ops
    box = None
    if ops_ and ops_[-1][0] == "crop":
        ops_, box = ops_[:-1], ops_[-1][1]
    if im is None and ops_:                    # a blank cell stays black through any resize
        ops_ = ()
    for op in ops_:
        im = resample.resize(im, op[1], op[2]) if op[0] == "resize" else resample.crop(im, op[1])
    w, h = cell.size
    ops.u8_to_model_input(im, box or (0, 0, w, h), out, col0)


class GridRequest(NamedTuple):
    """One request of ``VisualClozeModel.process_images_batch``: ``grid`` = (rows, cols), ``images`` / ``prompts`` / ``seed`` /
    ``cfg`` as ``set_grid_size(*grid)`` followed by ``process_images(images, prompts, seed, cfg)`` takes them."""
    grid: tuple
    images: list
    prompts: list
    seed: int = 0
    cfg: float = 30


def grid_tokens(cells, grid_h: int, grid_w: int) -> int:
    """Image tokens Li of a grid laid out by ``grid_plan``: every row is as high as its first cell and as wide as its cells together,
    one token per 16 x 16 pixels."""
    return sum(cells[i * grid_w].size[1] // 16 * sum(c.size[0] for c in cells[i * grid_w:(i + 1) * grid_w]) // 16 for i in range(grid_h))


def bucket_requests(token_counts, max_batch: int) -> list:
    """Which requests share a solve: indices with equal image-token counts (equal ``mu``, so equal schedules) go together, at most
    ``max_batch`` per solve; buckets come in order of their first request, requests keep their order inside a bucket.  Different
    counts never share a solve (nothing is padded).  Any hashable key works in place of a count (e.g. an image size)."""
    if isinstance(max_batch, bool) or not isinstance(max_batch, int) or max_batch < 1:
        raise ValueError(f"max_batch must be an int >= 1, got {max_batch!r}")
    groups = {}
    for i, n in enumerate(token_counts):
        groups.setdefault(n, []).append(i)
    return [idx[k:k + max_batch] for idx in groups.values() for k in range(0, len(idx), max_batch)]


# Default samples per batched solve by image-token count Li: (largest Li, batch), first match wins; beyond the last entry 1.
# Chosen from tools/bench_batch.py on an H100 (DESIGN.md §2g).
DEFAULT_MAX_BATCH = ((1152, 4),)


def default_max_batch(n_tokens: int) -> int:
    """The measured default of ``process_images_batch``'s ``max_batch`` for solves of ``n_tokens`` image tokens."""
    for top, b in DEFAULT_MAX_BATCH:
        if n_tokens <= top:
            return b
    return 1


def _sdedit_size(target_size) -> tuple:
    """(w, h) of the SDEdit solve for an output of ``target_size`` (None = 1024 x 1024): at most 1024 x 1024 pixels, aspect kept,
    both sides floored to multiples of 16 (visualcloze.py:163-175)."""
    if target_size is None:
        target_size = (1024, 1024)
    if target_size[0] * target_size[1] > 1024 * 1024:
        ar = target_size[0] / target_size[1]
        new_h = int((1024 * 1024 / ar) ** 0.5)
        target_size = (int(new_h * ar), new_h)
    return (target_size[0] // 16) * 16, (target_size[1] // 16) * 16


def _strip_content_prefix(content_prompt: str) -> str:
    """The content prompt of the SDEdit stage: the grid prompt's lead-in phrases removed (visualcloze.py:156-158)."""
    for c in _CONTENT_PREFIXES:
        if content_prompt.startswith(c):
            content_prompt = content_prompt.replace(c, "")
    return content_prompt


def _load_file(path: str, device) -> dict:
    """safetensors (BFL / diffusers releases) or a torch checkpoint (the LoRA files written by train.py:690-705)."""
    if str(path).endswith(".safetensors"):
        from safetensors.torch import load_file
        return load_file(path, device=str(device))
    return torch.load(path, map_location=device)


def _expand_state_dict(model, sd: dict) -> dict:
    """``optionally_expand_state_dict`` (models/util.py:456-472): zero-expand tensors smaller than the model's parameter
    (FLUX.1-dev ``img_in`` 64 -> 384 input channels when a non-Fill base is given)."""
    own = dict(model.named_parameters())
    for name, t in list(sd.items()):
        p = own.get(name)
        if p is not None and tuple(t.shape) != tuple(p.shape):
            big = torch.zeros_like(p, device=t.device)
            big[tuple(slice(0, d) for d in t.shape)] = t
            sd[name] = big
    return sd


class VisualClozeModel:
    def __init__(self, model_path=None, model_name="flux-dev-fill-lora", max_length=512, lora_rank=256, atol=1e-6, rtol=1e-3,
                 solver="euler", time_shifting_factor=1, resolution=384, precision="bf16", *, model=None, ae_decoder=None,
                 ae_encoder=None, t5=None, clip=None, encode=None, device=None, flux_ckpt=None, ae_ckpt=None, lora_mode="merged",
                 first_block_cache=None):
        """Positional arguments as the reference (visualcloze.py:79-82).  The reference constructor also pulls the base
        FLUX.1-Fill-dev weights (``load_flow_model``: ``$FLUX_DEV_FILL`` or a hub download) and the FLUX VAE
        (``AutoencoderKL.from_pretrained``); there is no network on the inference box, so here they come from files:
        ``flux_ckpt`` (default ``$FLUX_DEV_FILL``, BFL safetensors or a torch file) and ``ae_ckpt`` (default ``$AE``; BFL
        ``ae.safetensors`` or diffusers ``vae/diffusion_pytorch_model.safetensors`` -- keys are converted).  Pre-built
        ``model`` / ``ae_decoder`` / ``ae_encoder`` objects are used as they are.  Nothing is ever run on never-loaded
        parameters: the engines refuse to pack them.  ``lora_mode``: "merged" (default) or "unmerged", set on the flow model
        built or given (``FluxLoraWrapper.set_lora_mode``).  ``first_block_cache``: None (default, off) or the threshold of the
        opt-in first-block cache (``Flux.enable_first_block_cache``), set on the flow model likewise; the grid solve and the
        SDEdit solve each start it afresh."""
        if precision != "bf16":
            raise NotImplementedError("the sm_90a kernels implement the reference's default bf16 path only")
        if model_name != "flux-dev-fill-lora":
            raise NotImplementedError("VisualCloze uses the flux-dev-fill-lora geometry (models/util.py:132-165)")
        self.atol, self.rtol, self.solver = atol, rtol, solver
        self.time_shifting_factor, self.resolution, self.precision = time_shifting_factor, resolution, precision
        self.max_length, self.lora_rank = max_length, lora_rank
        self.device = torch.device(device if device is not None else "cuda")
        self.dtype = torch.bfloat16
        import os
        flux_ckpt = flux_ckpt or os.getenv("FLUX_DEV_FILL")
        ae_ckpt = ae_ckpt or os.getenv("AE")
        if model is None:
            with torch.device(self.device):
                model = FluxLoraWrapper(lora_rank=lora_rank, params=flux_dev_fill_params())
            if flux_ckpt is not None:                               # load_flow_model (models/util.py:406-411)
                sd = _expand_state_dict(model, _load_file(flux_ckpt, self.device))
                res = model.load_state_dict(sd, strict=False)
                if res.unexpected_keys:
                    raise ValueError(f"{flux_ckpt}: {len(res.unexpected_keys)} keys do not belong to the flux-dev-fill geometry, "
                                     f"e.g. {res.unexpected_keys[:3]}")
                del sd
        model.set_lora_mode(lora_mode)
        model.enable_first_block_cache(first_block_cache)
        self.model = model
        if model_path is not None:
            ckpt = _load_file(model_path, self.device)
            res = self.model.load_state_dict(ckpt, strict=False)    # LoRA tensors on top of the base (visualcloze.py:111-112)
            if res.unexpected_keys:
                raise ValueError(f"{model_path}: unexpected keys, e.g. {res.unexpected_keys[:3]}")
            del ckpt
        ae_sd = _load_file(ae_ckpt, self.device) if ae_ckpt is not None and (ae_decoder is None or (ae_encoder is None and encode is None)) else None
        if ae_decoder is None:
            with torch.device(self.device):
                ae_decoder = AutoEncoderDecoder()
            if ae_sd is not None:
                ae_decoder.load_state_dict(ae_sd, strict=True)
        self.ae = ae_decoder
        if ae_encoder is None and encode is None:
            with torch.device(self.device):
                ae_encoder = AutoEncoderEncoder()
            if ae_sd is not None:
                ae_encoder.load_state_dict(ae_sd, strict=True)
        self.ae_encoder = ae_encoder
        # fail at construction, not at the first image: a drop-in constructor must not leave torch.empty weights behind
        for what, mod in (("FLUX.1-Fill base weights (flux_ckpt= / $FLUX_DEV_FILL)", self.model), ("VAE decoder (ae_ckpt= / $AE)", self.ae),
                          ("VAE encoder (ae_ckpt= / $AE, or pass encode=)", self.ae_encoder)):
            missing = mod.uninitialized() if (mod is not None and hasattr(mod, "uninitialized")) else []
            if missing:
                raise RuntimeError(f"VisualClozeModel: {what}: {len(missing)} parameters were never loaded (e.g. {missing[:3]})")
        self.t5, self.clip, self.encode = t5, clip, encode
        self.sampler = Sampler(create_transport("Linear", "velocity", do_shift=True))
        self.sample_fn = self._make_sample_fn(30, True, self.time_shifting_factor, None)
        self.image_transform = image_transform
        self.grid_h = None
        self.grid_w = None

    def _make_sample_fn(self, num_steps, do_shift, tsf, strength):
        return self.sampler.sample_ode(sampling_method=self.solver, num_steps=num_steps, atol=self.atol, rtol=self.rtol,
                                       reverse=False, do_shift=do_shift, time_shifting_factor=tsf, strength=strength)

    def set_grid_size(self, h, w):
        self.grid_h, self.grid_w = h, w

    def _need(self, what):
        fn = getattr(self, what)
        if fn is None:
            raise RuntimeError(f"VisualClozeModel needs a `{what}` callable (text encoders and the VAE encoder are outside the "
                               "hot path; pass the reference's own, see the module docstring)")
        return fn

    def _encode_tokens(self, image_chw: torch.Tensor) -> torch.Tensor:
        """patchify((ae.encode(x).latent_dist.sample() - shift) * scale) in bf16 (visualcloze.py:377-378,384-385): [1, hw/256, 64].
        Like the reference, the sampling noise comes from the global (unseeded) RNG."""
        if self.encode is not None:
            lat = self.encode(image_chw[None].to(self.device, self.dtype))
            return _patchify(((lat - self.ae.shift_factor) * self.ae.scale_factor).to(self.dtype))
        x = image_chw[None].to(self.device)
        noise = torch.randn(1, self.ae_encoder.params.z_channels, x.shape[2] // 8, x.shape[3] // 8, device=self.device)
        return self.ae_encoder.encode_packed(x, noise)

    # ------------------------------------------------------------------------------------------------
    def _prepare_grid(self, images):
        """Resize / crop every cell to its row's reference size; blank + mask for the missing targets of the last row
        (visualcloze.py:300-360), with Pillow on the host.  -> (cells as PIL images, mask_position, upsampling_size)."""
        sizes = [[None if im is None else im.size for im in row] for row in images]
        cells, mask_position, upsampling_size = grid_plan(sizes, self.grid_h, self.grid_w, self.resolution)
        processed = [run_cell_pil(images[k // self.grid_w][k % self.grid_w], c) for k, c in enumerate(cells)]
        return processed, mask_position, upsampling_size

    def _grid_rows(self, images, grid=None):
        """The model input of every grid row built on the device, bit-identical to ``torch.cat([image_transform(c) for c in
        row], dim=2)`` over the cells of ``_prepare_grid``: each RGB image is uploaded once, resampled by libvcb200's Pillow
        resampler and written straight into its row.  ``grid``: (rows, cols), default ``set_grid_size``'s.
        -> (rows: fp32 [3, h, W] on the device, mask_position, upsampling_size)."""
        grid_h, grid_w = grid or (self.grid_h, self.grid_w)
        sizes = [[None if im is None else im.size for im in row] for row in images]
        cells, mask_position, upsampling_size = grid_plan(sizes, grid_h, grid_w, self.resolution)
        rows = []
        for i in range(grid_h):
            plans = cells[i * grid_w:(i + 1) * grid_w]
            widths = [c.size[0] for c in plans]
            row = torch.empty(3, plans[0].size[1], sum(widths), dtype=torch.float32, device=self.device)
            col = 0
            for j, cell in enumerate(plans):
                image = None if images[i][j] is None else resample.upload(images[i][j], self.device)
                run_cell_device(image, cell, row, col)
                col += widths[j]
            rows.append(row)
        return rows, mask_position, upsampling_size

    def _sdedit_resize(self, tile: torch.Tensor, box, size) -> torch.Tensor:
        """The SDEdit input image: the ``box`` crop of a uint8 [H, W, 3] device image, resized with BICUBIC to ``size``, on
        the device (``image.crop(box).resize(size)``)."""
        return resample.resize(resample.crop(tile, box), size, resample.BICUBIC)

    @torch.no_grad()
    def process_images(self, images, prompts, seed: int = 0, cfg: int = 30, steps: int = 30, upsampling_steps: int = 10,
                       upsampling_noise: float = 0.4, is_upsampling: bool = True):
        if seed == 0:
            seed = random.randint(0, 2 ** 32 - 1)
        self.sample_fn = self._make_sample_fn(int(steps), True, self.time_shifting_factor, None)
        grid_h, grid_w = self.grid_h, self.grid_w
        for i in range(grid_h):
            images[i] = [im.convert("RGB") if im is not None else None for im in images[i]]
        rows, mask_position, upsampling_size = self._grid_rows(images)

        dev, dt = self.device, self.dtype
        fill_mask = []
        for i, r in enumerate(rows):
            h, w = r.shape[1], r.shape[2] // grid_w
            marks = mask_position if i == grid_h - 1 else [0] * grid_w
            fill_mask.append(torch.cat([torch.full((1, 1, h, w), float(m), device=dev) for m in marks], dim=3))
        fill_cond = torch.cat([self._encode_tokens(r) for r in rows], dim=1)
        fill_mask = torch.cat([_pack_mask(m) for m in fill_mask], dim=1).to(dt)
        img_cond = torch.cat((fill_cond, fill_mask), dim=-1)

        rng = torch.Generator(device=dev).manual_seed(int(seed))
        noise, sizes = [], []
        for r in rows:
            h, w = r.shape[-2:]
            sizes.append((h, w))
            noise.append(torch.randn([1, 16, h // 8, w // 8], device=dev, generator=rng).to(dt))
        inp = prepare_modified(t5=self._need("t5"), clip=self._need("clip"), img=[noise], prompt=[" ".join(prompts)],
                               proportion_empty_prompts=0.0)
        kw = dict(txt=inp["txt"], txt_ids=inp["txt_ids"], txt_mask=inp["txt_mask"], y=inp["vec"], img_ids=inp["img_ids"],
                  img_mask=inp["img_mask"], cond=img_cond, guidance=torch.full((1,), cfg, device=dev, dtype=dt))
        samples = self.sample_fn(inp["img"], self.model.forward, kw)[-1][:1]

        # decode the query row only (the reference decodes all rows and crops the last, visualcloze.py:420-453)
        qh, qw = sizes[-1]
        n_tok = qh * qw // 256
        start = sum(h * w // 256 for h, w in sizes[:-1])
        tile = self.ae.decode_packed(samples[:, start:start + n_tok, :], qh // 16, qw // 16)[0]     # uint8 [3, H, W]
        tile = tile.permute(1, 2, 0).contiguous()                                                      # uint8 [H, W, 3]
        query = None if is_upsampling else Image.fromarray(tile.cpu().numpy())
        torch.cuda.empty_cache()

        ret = []
        ret_h, ret_w = tile.shape[0], tile.shape[1]
        for j in range(grid_w):
            if not mask_position[j]:
                continue
            box = (j * ret_w // grid_w, 0, (j + 1) * ret_w // grid_w, ret_h)
            if is_upsampling:
                ret.append(self._upsampling(tile, box, upsampling_size, cfg, upsampling_steps, upsampling_noise, rng, prompts[2]))
            else:
                ret.append(query.crop(box))
        return ret

    @torch.no_grad()
    def upsampling(self, image, target_size, cfg, upsampling_steps, upsampling_noise, generator, content_prompt):
        """SDEdit second stage (visualcloze.py:147-245): noise the resized image to `upsampling_noise`, denoise with an
        all-ones fill mask over a blank condition, 1x1 grid.  ``image`` (PIL; a mode other than RGB is converted as
        ``image_transform`` converts it) is uploaded once; the resize and the model input are made on the device."""
        if image.mode != "RGB":
            image = to_rgb_if_rgba(image).convert("RGB")
        return self._upsampling(resample.upload(image, self.device), (0, 0, image.width, image.height), target_size, cfg,
                                upsampling_steps, upsampling_noise, generator, content_prompt)

    def _upsampling(self, tile, box, target_size, cfg, upsampling_steps, upsampling_noise, generator, content_prompt):
        """``upsampling`` of the ``box`` crop of a uint8 [H, W, 3] device image."""
        content_prompt = _strip_content_prefix(content_prompt)
        size = _sdedit_size(target_size)
        image = self._sdedit_resize(tile, box, size)
        if upsampling_noise >= 1.0:
            return Image.fromarray(image.cpu().numpy())
        self.sample_fn = self._make_sample_fn(int(upsampling_steps), False, 1.0, upsampling_noise)
        dev, dt = self.device, self.dtype
        x = ops.u8_to_model_input(image, (0, 0) + size, torch.empty(3, size[1], size[0], dtype=torch.float32, device=dev), 0)
        latent = self._encode_tokens(x)
        blank = self._encode_tokens(torch.zeros_like(x))
        lh, lw = x.shape[1] // 8, x.shape[2] // 8
        mask = _pack_mask(torch.ones(1, 1, x.shape[1], x.shape[2], device=dev, dtype=dt))
        img_cond = torch.cat((blank, mask), dim=-1)
        noise = torch.randn([1, 16, lh, lw], device=dev, generator=generator).to(dt)
        inp = prepare_modified(t5=self._need("t5"), clip=self._need("clip"), img=[[noise]], prompt=[content_prompt],
                               proportion_empty_prompts=0.0)
        x_t = (inp["img"] * (1 - upsampling_noise) + latent * upsampling_noise).to(dt)
        kw = dict(txt=inp["txt"], txt_ids=inp["txt_ids"], txt_mask=inp["txt_mask"], y=inp["vec"], img_ids=inp["img_ids"],
                  img_mask=inp["img_mask"], cond=img_cond, guidance=torch.full((1,), cfg, device=dev, dtype=dt))
        sample = self.sample_fn(x_t, self.model.forward, kw)[-1][:1]
        tile = self.ae.decode_packed(sample, lh // 2, lw // 2)[0]
        return Image.fromarray(tile.permute(1, 2, 0).cpu().numpy())

    # ---- batched requests ----------------------------------------------------------------------------
    def _batch_size(self, n_tokens: int, n_evals: int, max_batch) -> int:
        """Samples per solve of ``n_tokens`` image tokens: ``max_batch`` (default: ``default_max_batch``), lowered until the
        engine's workspace for that batch fits in free device memory with 2 GiB to spare."""
        want = default_max_batch(n_tokens) if max_batch is None else max_batch
        if isinstance(want, bool) or not isinstance(want, int) or want < 1:
            raise ValueError(f"max_batch must be None or an int >= 1, got {max_batch!r}")
        if want == 1:
            return 1
        eng = self.model.engine()
        free = torch.cuda.mem_get_info(self.device)[0] + (eng._ws.numel() if eng._ws is not None else 0) - (2 << 30)
        while want > 1 and eng.lib.vcb_flux_workspace_bytes(eng._h, want, n_tokens, self.max_length, n_evals) > free:
            want -= 1
        return want

    def _n_evals(self, steps: int) -> int:
        from .ops import ODE_STAGES
        return ODE_STAGES[self.solver] * (int(steps) - 1)

    def _solve_batch(self, noise, prompts, conds, cfgs, sample_fn, blend=None):
        """One sampler solve of B samples with equal image-token counts: ``noise`` [per sample: list of row noises], ``prompts``
        [B] str, ``conds`` [B] tensors [1, Li, C], ``cfgs`` [B] guidance.  ``blend`` = (latents [B, Li, 64], s): start from
        ``noise * (1 - s) + latent * s`` (SDEdit).  -> final latent tokens [B, Li, 64]."""
        dev, dt = self.device, self.dtype
        inp = prepare_modified(t5=self._need("t5"), clip=self._need("clip"), img=noise, prompt=list(prompts), proportion_empty_prompts=0.0)
        x = inp["img"]
        if blend is not None:
            x = (x * (1 - blend[1]) + blend[0] * blend[1]).to(dt)
        kw = dict(txt=inp["txt"], txt_ids=inp["txt_ids"], txt_mask=inp["txt_mask"], y=inp["vec"], img_ids=inp["img_ids"],
                  img_mask=inp["img_mask"], cond=torch.cat(conds, dim=0),
                  guidance=torch.tensor([float(c) for c in cfgs], device=dev).to(dt))
        return sample_fn(x, self.model.forward, kw)[-1][:len(prompts)]

    def _decode_groups(self, items, max_batch: int) -> list:
        """items: (tokens [Li, 64], h, w) -> uint8 [3, 16h, 16w] per item; equal sizes share ``decode_packed`` calls of up to
        ``max_batch`` images, fewer when the decoder's workspace for them would not fit in free memory with 2 GiB to spare."""
        out = [None] * len(items)
        for size in dict.fromkeys((h, w) for _, h, w in items):
            idx = [k for k, it in enumerate(items) if it[1:] == size]
            n = min(max_batch, len(idx))
            if n > 1 and hasattr(self.ae, "_engine"):
                lib, hnd = _vcb_lib.lib(), self.ae._engine()
                free = torch.cuda.mem_get_info(self.device)[0] + (self.ae._ws.numel() if self.ae._ws is not None else 0) - (2 << 30)
                while n > 1 and lib.vcb_vae_workspace_bytes(hnd, n, *size) > free:
                    n -= 1
            for chunk in bucket_requests([size] * len(idx), n):
                tiles = self.ae.decode_packed(torch.stack([items[idx[k]][0] for k in chunk]), *size)
                for j, k in enumerate(chunk):
                    out[idx[k]] = tiles[j]
        return out

    @torch.no_grad()
    def process_images_batch(self, requests, *, steps: int = 30, upsampling_steps: int = 10, upsampling_noise: float = 0.4,
                             is_upsampling: bool = True, max_batch: int | None = None) -> list:
        """Several grids in batched solves.  ``requests``: ``GridRequest``s (or dicts of their fields).  Returns one list of PIL
        images per request, each what ``set_grid_size(*grid)`` followed by ``process_images(images, prompts, seed, cfg, steps,
        upsampling_steps, upsampling_noise, is_upsampling)`` returns (within the bf16 batch-invariance of the kernels).

        Requests with the same image-token count share one solve of up to ``max_batch`` samples (None: ``default_max_batch``,
        lowered to what device memory holds); different counts run apart, nothing is padded.  Every request draws its noise from
        its own ``torch.Generator(device).manual_seed(seed)`` in the solo order (grid rows, then one SDEdit noise per target in
        column order); ``seed == 0`` draws a random seed per request.  SDEdit targets of all requests are batched by their own
        token count.  With the first-block cache on, batched solves decide per sample.  ``set_grid_size`` is left as it was."""
        reqs = [r if isinstance(r, GridRequest) else GridRequest(**r) for r in requests]
        dev, dt = self.device, self.dtype
        fbc, fbc_per_sample = getattr(self.model, "_fbc", 0.0), getattr(self.model, "_fbc_per_sample", False)
        if fbc > 0 and not fbc_per_sample:
            self.model.enable_first_block_cache(fbc, per_sample=True)
        try:
            return self._process_batch(reqs, int(steps), int(upsampling_steps), float(upsampling_noise), is_upsampling, max_batch, dev, dt)
        finally:
            if fbc > 0 and not fbc_per_sample:
                self.model.enable_first_block_cache(fbc, per_sample=False)

    def _process_batch(self, reqs, steps, upsampling_steps, upsampling_noise, is_upsampling, max_batch, dev, dt):
        preps = []
        for r in reqs:
            grid_h, grid_w = (int(v) for v in r.grid)
            seed = r.seed if r.seed != 0 else random.randint(0, 2 ** 32 - 1)
            images = [[im.convert("RGB") if im is not None else None for im in row] for row in r.images]
            rows, mask_position, upsampling_size = self._grid_rows(images, (grid_h, grid_w))
            fill_mask = []
            for i, row in enumerate(rows):
                h, w = row.shape[1], row.shape[2] // grid_w
                marks = mask_position if i == grid_h - 1 else [0] * grid_w
                fill_mask.append(torch.cat([torch.full((1, 1, h, w), float(m), device=dev) for m in marks], dim=3))
            fill_cond = torch.cat([self._encode_tokens(row) for row in rows], dim=1)
            fill_mask = torch.cat([_pack_mask(m) for m in fill_mask], dim=1).to(dt)
            rng = torch.Generator(device=dev).manual_seed(int(seed))
            sizes = [tuple(row.shape[-2:]) for row in rows]
            noise = [torch.randn([1, 16, h // 8, w // 8], device=dev, generator=rng).to(dt) for h, w in sizes]
            preps.append(dict(grid_w=grid_w, mask_position=mask_position, upsampling_size=upsampling_size, rng=rng, sizes=sizes,
                              noise=noise, cond=torch.cat((fill_cond, fill_mask), dim=-1), Li=sum(h * w // 256 for h, w in sizes)))

        # grid solves: one per bucket of equal Li
        n_evals = self._n_evals(steps)
        samples = [None] * len(reqs)
        for Li in dict.fromkeys(p["Li"] for p in preps):
            idx = [k for k, p in enumerate(preps) if p["Li"] == Li]
            for bucket in bucket_requests([Li] * len(idx), self._batch_size(Li, n_evals, max_batch)):
                ks = [idx[k] for k in bucket]
                out = self._solve_batch([preps[k]["noise"] for k in ks], [" ".join(reqs[k].prompts) for k in ks],
                                        [preps[k]["cond"] for k in ks], [reqs[k].cfg for k in ks],
                                        self._make_sample_fn(steps, True, self.time_shifting_factor, None))
                for n, k in enumerate(ks):
                    samples[k] = out[n]

        # decode the query rows, equal sizes together
        items = []
        for p, smp in zip(preps, samples):
            qh, qw = p["sizes"][-1]
            start = sum(h * w // 256 for h, w in p["sizes"][:-1])
            items.append((smp[start:start + qh * qw // 256], qh // 16, qw // 16))
        tiles = self._decode_groups(items, self._batch_size(max(p["Li"] for p in preps), n_evals, max_batch))
        tiles = [t.permute(1, 2, 0).contiguous() for t in tiles]                                  # uint8 [H, W, 3]

        results, targets = [[] for _ in reqs], []
        for k, (p, tile) in enumerate(zip(preps, tiles)):
            ret_h, ret_w = tile.shape[0], tile.shape[1]
            query = None if is_upsampling else Image.fromarray(tile.cpu().numpy())
            for j in range(p["grid_w"]):
                if not p["mask_position"][j]:
                    continue
                box = (j * ret_w // p["grid_w"], 0, (j + 1) * ret_w // p["grid_w"], ret_h)
                if not is_upsampling:
                    results[k].append(query.crop(box))
                    continue
                size = _sdedit_size(p["upsampling_size"])
                image = self._sdedit_resize(tile, box, size)
                if upsampling_noise >= 1.0:
                    results[k].append(Image.fromarray(image.cpu().numpy()))
                    continue
                x = ops.u8_to_model_input(image, (0, 0) + size, torch.empty(3, size[1], size[0], dtype=torch.float32, device=dev), 0)
                latent = self._encode_tokens(x)
                blank = self._encode_tokens(torch.zeros_like(x))
                mask = _pack_mask(torch.ones(1, 1, x.shape[1], x.shape[2], device=dev, dtype=dt))
                noise = torch.randn([1, 16, x.shape[1] // 8, x.shape[2] // 8], device=dev, generator=p["rng"]).to(dt)
                results[k].append(None)
                targets.append(dict(req=k, slot=len(results[k]) - 1, size=size, latent=latent, cond=torch.cat((blank, mask), dim=-1),
                                    noise=noise, cfg=reqs[k].cfg, prompt=_strip_content_prefix(reqs[k].prompts[2])))
        if not targets:
            return results

        # SDEdit solves: targets batched by their own token count
        n_evals = self._n_evals(upsampling_steps)
        lats = [None] * len(targets)
        for Li in dict.fromkeys(t["size"][0] * t["size"][1] // 256 for t in targets):
            idx = [k for k, t in enumerate(targets) if t["size"][0] * t["size"][1] // 256 == Li]
            for bucket in bucket_requests([Li] * len(idx), self._batch_size(Li, n_evals, max_batch)):
                ts = [targets[idx[k]] for k in bucket]
                out = self._solve_batch([[t["noise"]] for t in ts], [t["prompt"] for t in ts], [t["cond"] for t in ts],
                                        [t["cfg"] for t in ts], self._make_sample_fn(upsampling_steps, False, 1.0, upsampling_noise),
                                        blend=(torch.cat([t["latent"] for t in ts], dim=0), upsampling_noise))
                for n, k in enumerate(bucket):
                    lats[idx[k]] = out[n]
        tiles = self._decode_groups([(lat, t["size"][1] // 16, t["size"][0] // 16) for lat, t in zip(lats, targets)],
                                    self._batch_size(max(t["size"][0] * t["size"][1] // 256 for t in targets), n_evals, max_batch))
        for t, tile in zip(targets, tiles):
            results[t["req"]][t["slot"]] = Image.fromarray(tile.permute(1, 2, 0).cpu().numpy())
        return results
