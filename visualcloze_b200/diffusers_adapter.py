"""``VisualClozePipeline``-shaped front end (the diffusers pipeline the reference's README points to, README.md:141-205) over
``VisualClozeModel`` -- the caller on the far side of the hot path (SURVEY.md 8f-4).

The diffusers pipeline is not part of /root/reference (README.md:143 links it); what is mirrored here is its documented call:

    pipe(task_prompt=..., content_prompt=..., image=[[...], [..., None]], upsampling_height=..., upsampling_width=...,
         upsampling_strength=..., guidance_scale=30, num_inference_steps=30, max_sequence_length=512, generator=...).images[0][0]

mapped onto the reference's own entry (visualcloze.py:247-467): ``image`` is the grid (rows of PIL images, ``None`` = target),
the layout prompt is the first template of ``get_layout_instruction`` (data/prefix_instruction.py:684-697, what app.py:116
pre-fills: "A grid layout with R rows and C columns, displaying N images arranged side by side."), ``upsampling_strength`` is the SDEdit
noise level, ``generator`` supplies the seed.  Text encoders / VAE weights are whatever the wrapped ``VisualClozeModel`` holds.
"""
from __future__ import annotations

from dataclasses import dataclass, field

import torch


@dataclass
class PipelineOutput:
    images: list = field(default_factory=list)          # [sample][target] PIL images, like the diffusers pipeline output


def layout_prompt(rows: int, cols: int) -> str:
    """first template of the reference's ``get_layout_instruction(cols, rows)`` (data/prefix_instruction.py:686)"""
    return f"A grid layout with {rows} rows and {cols} columns, displaying {rows * cols} images arranged side by side."


def _is_grid(x) -> bool:
    """a grid is a list of rows whose entries are images or None; a list of grids has lists one level deeper"""
    return isinstance(x, list) and bool(x) and all(isinstance(r, list) for r in x) and not any(isinstance(c, list) for r in x for c in r)


def _check_grid(image) -> int:
    if not _is_grid(image):
        raise ValueError("image must be a list of rows (lists of PIL images; None marks a target in the last row), or a list of such grids")
    cols = len(image[0])
    if any(len(r) != cols for r in image):
        raise ValueError("every grid row needs the same number of images")
    if any(im is None for r in image[:-1] for im in r):
        raise ValueError("Please provide each image in the in-context example.")
    return cols


def _as_list(value, what: str, n: int) -> list:
    """one value for every prompt, or a list of n"""
    if not isinstance(value, list):
        return [value] * n
    if len(value) != n:
        raise ValueError(f"{what}: {len(value)} entries for {n} prompts")
    return value


def request_seeds(generator, n_images: int) -> list:
    """Seeds of ``n_images`` images: no generator -> 0 each (a random seed per image); one generator with seed s -> s, s + 1, ...;
    a list of generators -> one seed per image, its ``initial_seed()``."""
    if isinstance(generator, (list, tuple)):
        if len(generator) != n_images:
            raise ValueError(f"{len(generator)} generators for {n_images} images: pass one per image, or a single one")
        return [int(g.initial_seed()) for g in generator]
    if generator is None:
        return [0] * n_images
    s = int(generator.initial_seed())
    return [s + k for k in range(n_images)]


class VisualClozePipelineAdapter:
    def __init__(self, model):
        self.model = model                                # a visualcloze_b200.pipeline.VisualClozeModel

    @torch.no_grad()
    def __call__(self, task_prompt, content_prompt, image: list, upsampling_height: int | None = None,
                 upsampling_width: int | None = None, upsampling_strength: float = 0.4, guidance_scale: float = 30.0,
                 num_inference_steps: int = 30, upsampling_steps: int = 10, max_sequence_length: int = 512, generator=None,
                 num_images_per_prompt: int = 1, max_batch: int | None = None, **unused) -> PipelineOutput:
        """Like the diffusers pipeline: ``task_prompt`` / ``content_prompt`` / ``image`` may each be one value or a list with one
        entry per prompt (``image``: one grid or a list of grids), and each prompt gives ``num_images_per_prompt`` images.
        ``images`` of the output has one list of target images per image made, prompt by prompt.  Seeds: a single ``generator``
        with seed s gives the images seeds s, s + 1, ... in that order; a list of generators (one per image) gives each image the
        seed of its own; none gives every image a random seed.  More than one image runs through
        ``VisualClozeModel.process_images_batch`` (``max_batch`` goes there); one image is one ``process_images`` call."""
        if max_sequence_length != self.model.max_length:
            raise ValueError(f"the wrapped model was built for max_length={self.model.max_length}")
        if isinstance(num_images_per_prompt, bool) or not isinstance(num_images_per_prompt, int) or num_images_per_prompt < 1:
            raise ValueError(f"num_images_per_prompt must be an int >= 1, got {num_images_per_prompt!r}")
        grids = [image] if _is_grid(image) else image
        if not isinstance(grids, list) or not grids:
            raise ValueError("image must be a list of rows (lists of PIL images; None marks a target in the last row), or a list of such grids")
        n = max(len(v) for v in (task_prompt, content_prompt, grids) if isinstance(v, list))
        grids = _as_list(grids, "image", n) if len(grids) > 1 else grids * n
        tasks, contents = _as_list(task_prompt, "task_prompt", n), _as_list(content_prompt, "content_prompt", n)
        for g in grids:
            _check_grid(g)
        seeds = request_seeds(generator, n * num_images_per_prompt)
        is_up = upsampling_strength < 1.0 and (upsampling_height is not None or upsampling_width is not None)
        kw = dict(steps=int(num_inference_steps), upsampling_steps=int(upsampling_steps), upsampling_noise=float(upsampling_strength),
                  is_upsampling=is_up)
        reqs = []
        for p in range(n):
            prompts = [layout_prompt(len(grids[p]), len(grids[p][0])), tasks[p] or "", contents[p] or ""]
            for i in range(num_images_per_prompt):
                reqs.append(dict(grid=(len(grids[p]), len(grids[p][0])), images=[list(r) for r in grids[p]], prompts=prompts,
                                 seed=seeds[p * num_images_per_prompt + i], cfg=guidance_scale))
        if len(reqs) == 1:
            r = reqs[0]
            self.model.set_grid_size(*r["grid"])
            outs = [self.model.process_images(r["images"], r["prompts"], seed=r["seed"], cfg=r["cfg"], **kw)]
        else:
            outs = self.model.process_images_batch(reqs, max_batch=max_batch, **kw)
        if is_up and upsampling_height and upsampling_width:
            outs = [[im.resize((int(upsampling_width) // 16 * 16, int(upsampling_height) // 16 * 16)) if im.size != (upsampling_width, upsampling_height) else im
                     for im in out] for out in outs]
        return PipelineOutput(images=outs)
