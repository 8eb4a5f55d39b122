"""Context number, NOT part of the product or of bench.py: the reference's algorithm (oracle port, un-merged LoRA r=256,
bf16 autocast semantics) executed EAGERLY ON THE GPU with library kernels -- cuBLAS GEMMs, ATen elementwise ops and the
same flash-attn 2.x kernel the reference calls (models/math.py:85-95) -- on the cfg-B shapes.  It approximates what the
unmodified reference costs per model evaluation on this H100 (the reference itself is not part of this repository).

    python tests/perf_reference_gpu.py [n_double n_single]      -> one JSON line, extrapolated to 19 + 38 blocks
"""
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import flux_oracle as fo  # noqa: E402

try:
    from flash_attn import flash_attn_func
except Exception:  # noqa: BLE001
    flash_attn_func = None


def fa2_attention(q, k, v, cos, sin, mask, nm):
    q, k = fo.apply_rope(q, cos, sin), fo.apply_rope(k, cos, sin)
    B, H, L, D = q.shape
    o = flash_attn_func(q.transpose(1, 2), k.transpose(1, 2), v.transpose(1, 2))
    return o.reshape(B, L, H * D)


def main():
    nd, ns = (int(sys.argv[1]), int(sys.argv[2])) if len(sys.argv) > 2 else (2, 4)
    dev = "cuda"
    if flash_attn_func is not None:
        fo.joint_attention = fa2_attention
    cfg = fo.FluxConfig(depth=nd, depth_single_blocks=ns, lora_rank=256)
    shapes = fo.param_shapes(cfg)
    g = torch.Generator(device=dev).manual_seed(0)
    p = {}
    for k, shp in shapes.items():
        std = 0.02 if (k.endswith(".bias") or "lora_B" in k) else shp[-1] ** -0.5
        p[k] = torch.ones(shp, dtype=torch.bfloat16, device=dev) if k.endswith(".scale") else \
            (torch.randn(shp, generator=g, device=dev) * std).to(torch.bfloat16)
    Li, Lt = 3456, 512
    img = torch.randn(1, Li, 384, generator=g, device=dev).bfloat16()
    txt = (0.1 * torch.randn(1, Lt, 4096, generator=g, device=dev)).bfloat16()
    ids = torch.zeros(1, Li, 3, device=dev)
    ids[0, :, 0], ids[0, :, 1], ids[0, :, 2] = 1 + torch.arange(Li, device=dev) // 1728, (torch.arange(Li, device=dev) % 1728) // 72, torch.arange(Li, device=dev) % 72
    kw = dict(img=img, img_ids=ids, txt=txt, txt_ids=torch.zeros(1, Lt, 3, device=dev), timesteps=torch.tensor([0.7], device=dev),
              y=torch.randn(1, 768, generator=g, device=dev).bfloat16(), txt_mask=torch.ones(1, Lt, dtype=torch.int32, device=dev),
              img_mask=torch.ones(1, Li, dtype=torch.int32, device=dev), guidance=torch.full((1,), 30.0, dtype=torch.bfloat16, device=dev))

    def run(cfg_):
        with torch.no_grad():
            return fo.flux_forward(p, cfg_, **kw, mode="cuda_bf16")

    def timed(cfg_):
        for _ in range(2):
            run(cfg_)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(3):
            run(cfg_)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / 3

    import dataclasses
    t_full = timed(cfg)
    t_d = timed(dataclasses.replace(cfg, depth_single_blocks=0))
    t_0 = timed(dataclasses.replace(cfg, depth=0, depth_single_blocks=0))
    per_double = (t_d - t_0) / nd
    per_single = (t_full - t_d) / ns
    ms_eval = t_0 + 19 * per_double + 38 * per_single
    print(json.dumps({"what": "reference algorithm, eager torch on GPU (cuBLAS + ATen + FA2), un-merged LoRA, cfg B tokens",
                      "attention": "flash_attn 2.x" if flash_attn_func is not None else "explicit softmax",
                      "ms_per_double_block": per_double, "ms_per_single_block": per_single, "ms_embed_final": t_0,
                      "ms_per_evaluation_extrapolated": ms_eval, "images_per_s_29_evals": 1000.0 / (29 * ms_eval)}))


if __name__ == "__main__":
    main()
