"""Micro-benchmarks of the hot kernels on one H100 (CUDA events, L2 flushed between timed launches).
Prints one JSON line per case and writes gpurun_out/bench_kernels.jsonl.  Library kernels (cuBLAS via torch.matmul,
FA2, cuDNN/flash SDPA) are timed next to ours as reference points only; they are never on the product path."""
import json
import math
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from visualcloze_b200 import ops  # noqa: E402

BF16 = torch.bfloat16
dev = "cuda"
flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)
out_f = open("gpurun_out/bench_kernels.jsonl", "a")


def timeit(fn, iters=10, warm=3):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    ts.sort()
    return ts[len(ts) // 2], ts[0]


def emit(**kw):
    line = json.dumps(kw)
    print(line, flush=True)
    out_f.write(line + "\n")
    out_f.flush()


def bench_gemm(which):
    shapes = [("img_qkv", 3456, 9216, 3072), ("img_proj", 3456, 3072, 3072), ("img_mlp_up", 3456, 12288, 3072),
              ("img_mlp_down", 3456, 3072, 12288), ("sgl_linear1", 3968, 21504, 3072), ("sgl_linear2", 3968, 3072, 15360),
              ("txt_qkv", 512, 9216, 3072), ("mod_batched", 29, 18432, 3072), ("square8k", 8192, 8192, 8192)]
    for name, M, N, K in shapes:
        if which and which not in name:
            continue
        a = torch.randn(M, K, device=dev).to(BF16)
        w = (torch.randn(N, K, device=dev) / math.sqrt(K)).to(BF16)
        bias = torch.randn(N, device=dev)
        out = torch.empty(M, N, dtype=BF16, device=dev)
        fl = 2.0 * M * N * K
        med, best = timeit(lambda: torch.matmul(a, w.t()))
        emit(kernel="cublas", name=name, M=M, N=N, K=K, ms=med, tflops=fl / med / 1e9, best_tflops=fl / best / 1e9)
        for cg in (1, 2):
            for bn in (128, 192, 256):
                try:
                    med, best = timeit(lambda: ops.gemm(a, w, bias, out, block_n=bn, cta_group=cg))
                    emit(kernel="vcb_gemm", name=name, M=M, N=N, K=K, block_n=bn, cta_group=cg, ms=med,
                         tflops=fl / med / 1e9, best_tflops=fl / best / 1e9)
                except Exception as e:  # noqa: BLE001
                    emit(kernel="vcb_gemm", name=name, block_n=bn, cta_group=cg, error=str(e))


def bench_attn():
    heads = 24
    H = heads * 128
    for L in (1088, 3968, 5696, 7424):
        qkv = torch.randn(L, 3 * H, device=dev).to(BF16)
        out = torch.empty(L, H, dtype=BF16, device=dev)
        fl = 4.0 * L * L * H
        med, best = timeit(lambda: ops.attention(qkv, 1, L, heads, out, q_col=0, k_col=H, v_col=2 * H))
        emit(kernel="vcb_attention", L=L, ms=med, tflops=fl / med / 1e9, best_tflops=fl / best / 1e9)
        med, best = timeit(lambda: ops.attention(qkv, 1, L, heads, out, q_col=0, k_col=H, v_col=2 * H, score_bound_log2=30.0))
        emit(kernel="vcb_attention_bounded", L=L, ms=med, tflops=fl / med / 1e9, best_tflops=fl / best / 1e9)
        q, k, v = (qkv[:, i * H:(i + 1) * H].reshape(1, L, heads, 128) for i in range(3))
        try:
            from flash_attn import flash_attn_func
            med, best = timeit(lambda: flash_attn_func(q, k, v))
            emit(kernel="fa2_sm100", L=L, ms=med, tflops=fl / med / 1e9, best_tflops=fl / best / 1e9)
        except Exception as e:  # noqa: BLE001
            emit(kernel="fa2_sm100", L=L, error=str(e)[:200])
        qt, kt, vt = (t.transpose(1, 2) for t in (q, k, v))
        try:
            med, best = timeit(lambda: torch.nn.functional.scaled_dot_product_attention(qt, kt, vt))
            emit(kernel="torch_sdpa", L=L, ms=med, tflops=fl / med / 1e9, best_tflops=fl / best / 1e9)
        except Exception as e:  # noqa: BLE001
            emit(kernel="torch_sdpa", L=L, error=str(e)[:200])


def bench_ln():
    for rows in (3456, 3968):
        H = 3072
        x = torch.randn(rows, H, device=dev).to(BF16)
        sh, sc = torch.randn(1, H, device=dev).to(BF16), torch.randn(1, H, device=dev).to(BF16)
        out = torch.empty_like(x)
        med, best = timeit(lambda: ops.ln_modulate(x, sh, sc, out, rows_per_batch=rows))
        by = 4.0 * rows * H
        emit(kernel="vcb_ln_modulate", rows=rows, ms=med, gbs=by / med / 1e6, best_gbs=by / best / 1e6)


if __name__ == "__main__":
    what = sys.argv[1] if len(sys.argv) > 1 else "all"
    if what in ("all", "gemm"):
        bench_gemm(sys.argv[2] if len(sys.argv) > 2 else "")
    if what in ("all", "attn"):
        bench_attn()
    if what in ("all", "ln"):
        bench_ln()
