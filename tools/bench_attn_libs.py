"""Attention kernel vs the libraries on the reference's shapes (24 heads, head_dim 128, bf16), one H100.

  vcb  per-tile grid / persistent schedule  x  exact online-max / fixed-reference softmax
  cuDNN SDPA (torch.nn.functional.scaled_dot_product_attention, cudnn backend), flash-attn 2 (what models/math.py:85 calls)

CUDA events around each launch, L2 flushed between timed launches, median of 15.  Writes gpurun_out/attn_vs_libs.json.
Library kernels are reference points only -- they are never on the product path."""
import json
import math
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from visualcloze_b200 import ops  # noqa: E402

BF16 = torch.bfloat16
flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device="cuda")


def timeit(fn, iters=15, warm=3):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        flush.zero_()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); fn(); b.record(); torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    ts.sort()
    return ts[len(ts) // 2]


def sustained(fn, seconds=0.5):
    """back-to-back launches for `seconds`: the power-capped steady state the denoising loop runs in (no flush: K / V of one
    24-head call are 48 - 91 MB and the launches follow each other like the 57 attention calls of an evaluation do)"""
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record(); fn(); b.record(); torch.cuda.synchronize()
    n = max(10, int(seconds * 1e3 / max(a.elapsed_time(b), 1e-3)))
    a.record()
    for _ in range(n):
        fn()
    b.record(); torch.cuda.synchronize()
    return a.elapsed_time(b) / n


def main():
    heads, H = 24, 3072
    rows = []
    for L in (1088, 3968, 4608, 6656, 7424):
        g = torch.Generator(device="cuda").manual_seed(L)
        qkv = torch.randn(L, 3, heads, 128, generator=g, device="cuda")
        for i, a in ((0, 1.2), (1, 1.1)):
            qkv[:, i] = a * qkv[:, i] / qkv[:, i].pow(2).mean(-1, keepdim=True).sqrt()
        qkv = qkv.reshape(L, 3 * H).to(BF16)
        bound = 1.2 * 1.1 * math.sqrt(128.0) * math.log2(math.e) * 1.03
        out = torch.empty(L, H, dtype=BF16, device="cuda")
        fl = 4.0 * L * L * H
        rec = {"L": L, "heads": heads, "flops": fl}
        for sched, sname in ((1, "per_pair"), (2, "persistent")):
            for sb, bname in ((0.0, "exact"), (bound, "bounded")):
                f = lambda: ops.attention(qkv, 1, L, heads, out, q_col=0, k_col=H, v_col=2 * H, score_bound_log2=sb, schedule=sched)
                ms = timeit(f)
                ms_s = sustained(f)
                rec[f"vcb_{sname}_{bname}"] = {"us": ms * 1e3, "tflops": fl / ms / 1e9, "sustained_us": ms_s * 1e3, "sustained_tflops": fl / ms_s / 1e9}
        q, k, v = (qkv[:, i * H:(i + 1) * H].reshape(1, L, heads, 128) for i in range(3))
        qt, kt, vt = (t.transpose(1, 2).contiguous() for t in (q, k, v))
        try:
            from torch.nn.attention import SDPBackend, sdpa_kernel
            with sdpa_kernel(SDPBackend.CUDNN_ATTENTION):
                f = lambda: torch.nn.functional.scaled_dot_product_attention(qt, kt, vt)
                ms = timeit(f)
                ms_s = sustained(f)
            rec["cudnn_sdpa"] = {"us": ms * 1e3, "tflops": fl / ms / 1e9, "sustained_us": ms_s * 1e3, "sustained_tflops": fl / ms_s / 1e9}
        except Exception as e:  # noqa: BLE001
            rec["cudnn_sdpa"] = {"error": str(e)[:200]}
        try:
            from flash_attn import flash_attn_func
            qc, kc, vc = q.contiguous(), k.contiguous(), v.contiguous()
            f = lambda: flash_attn_func(qc, kc, vc)
            ms = timeit(f)
            ms_s = sustained(f, 0.3)
            rec["flash_attn2"] = {"us": ms * 1e3, "tflops": fl / ms / 1e9, "sustained_us": ms_s * 1e3, "sustained_tflops": fl / ms_s / 1e9}
        except Exception as e:  # noqa: BLE001
            rec["flash_attn2"] = {"error": str(e)[:200]}
        print(json.dumps(rec), flush=True)
        rows.append(rec)
    os.makedirs("gpurun_out", exist_ok=True)
    json.dump({"gpu": torch.cuda.get_device_name(0), "method": "us / tflops: CUDA events per launch, 256 MiB L2 flush between launches, median of 15 (burst clocks); "
               "sustained_*: back-to-back launches for 0.5 s, CUDA events around the run (power-capped steady state, as in the denoising loop)",
               "rows": rows}, open("gpurun_out/attn_vs_libs.json", "w"), indent=1)


if __name__ == "__main__":
    main()
