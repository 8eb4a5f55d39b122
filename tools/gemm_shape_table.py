"""Per-shape GEMM table for the cfg-B FLUX-DiT step: ours (real fused epilogue) vs cuBLAS (torch.matmul, no epilogue) on the same
shape, each run BACK TO BACK for ~0.6 s so the chip reaches the clocks it sustains in the denoising loop (a burst number says little).  CUDA events around the whole run; writes the table as JSON.
cuBLAS is a reference point only -- it is never on the product path."""
import json
import math
import os
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from visualcloze_b200 import ops  # noqa: E402

BF16 = torch.bfloat16
dev = "cuda"
H, MLP, Li, Lt = 3072, 12288, 3456, 512
L = Li + Lt


def sustained(fn, seconds=0.6):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    # calibrate
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record(); fn(); b.record(); torch.cuda.synchronize()
    n = max(10, int(seconds * 1e3 / max(a.elapsed_time(b), 1e-3)))
    a.record()
    for _ in range(n):
        fn()
    b.record(); torch.cuda.synchronize()
    return a.elapsed_time(b) / n


def main():
    g = torch.Generator(device=dev).manual_seed(0)
    rn = lambda *s: torch.randn(*s, generator=g, device=dev)
    rope = torch.zeros(64, L, 2, device=dev); rope[..., 0] = 1.0
    qs = torch.ones(128, dtype=BF16, device=dev)
    gate = (0.3 * rn(1, 6 * H)).to(BF16)
    rows = []
    # (name, grouped [(rows, row offset)], N, K, epilogue, count per evaluation)
    cases = [("double qkv (img+txt grouped)", [(Li, Lt), (Lt, 0)], 3 * H, H, "qkv", 19),
             ("double proj (grouped)", [(Li, Lt), (Lt, 0)], H, H, "gate_res", 19),
             ("double mlp.0 (grouped)", [(Li, Lt), (Lt, 0)], MLP, H, "gelu", 19),
             ("double mlp.2 (grouped)", [(Li, Lt), (Lt, 0)], H, MLP, "gate_res", 19),
             ("single linear1", [(L, 0)], 3 * H + MLP, H, "linear1", 38),
             ("single linear2", [(L, 0)], H, H + MLP, "gate_res", 38)]
    for name, parts, N, K, epi, count in cases:
        a = (rn(L, K)).to(BF16)
        x = rn(L, H).to(BF16)
        qkv = torch.empty(L, 3 * H, dtype=BF16, device=dev)
        cat = torch.empty(L, H + MLP, dtype=BF16, device=dev)
        ws = [(rn(N, K) / math.sqrt(K)).to(BF16) for _ in parts]
        bs = [rn(N) for _ in parts]
        probs = []
        for (r, off), w, b in zip(parts, ws, bs):
            kw = dict(a=a[off:off + r], w=w, bias=b, rows_per_batch=r, out_batch_rows=L, out_row_offset=off)
            if epi == "qkv":
                kw.update(out=qkv, epilogue=ops.EPI_QKV, hidden=H, q_scale=qs, k_scale=qs, rope=rope)
            elif epi == "linear1":
                kw.update(out=qkv, epilogue=ops.EPI_LINEAR1, hidden=H, q_scale=qs, k_scale=qs, rope=rope, out2=cat, out2_col_offset=H)
            elif epi == "gelu":
                kw.update(out=cat, epilogue=ops.EPI_BIAS_GELU, out_col_offset=H)
            else:
                kw.update(out=x, epilogue=ops.EPI_GATE_RES, gate=gate[:, :N], res=x)
            probs.append(kw)

        def ours():
            if len(probs) == 2:
                ops.gemm_grouped(probs[0], probs[1])
            else:
                d = dict(probs[0]); ops.gemm(d.pop("a"), d.pop("w"), d.pop("bias"), d.pop("out"), **d)

        outs = [torch.empty(r, N, dtype=BF16, device=dev) for r, _ in parts]

        def cublas():
            for (r, off), w, o in zip(parts, ws, outs):
                torch.matmul(a[off:off + r], w.t(), out=o)

        fl = sum(2.0 * r * N * K for r, _ in parts)
        t_o, t_c = sustained(ours), sustained(cublas)
        time.sleep(0.2)
        rec = dict(name=name, M=sum(r for r, _ in parts), N=N, K=K, epilogue=epi, per_eval=count, gflop=fl / 1e9,
                   ours_us=t_o * 1e3, ours_tflops=fl / t_o / 1e9, cublas_us=t_c * 1e3, cublas_tflops=fl / t_c / 1e9,
                   ours_over_cublas=t_c / t_o)
        print(json.dumps(rec), flush=True)
        rows.append(rec)
    tot_o = sum(r["ours_us"] * r["per_eval"] for r in rows)
    tot_c = sum(r["cublas_us"] * r["per_eval"] for r in rows)
    os.makedirs("gpurun_out", exist_ok=True)
    json.dump({"gpu": torch.cuda.get_device_name(0), "method": "back-to-back launches for ~0.6 s per shape (power-capped steady state), CUDA events",
               "rows": rows, "per_eval_ms": {"ours": tot_o / 1e3, "cublas_without_epilogues": tot_c / 1e3}}, open("gpurun_out/gemm_shapes.json", "w"), indent=1)
    print("per evaluation: ours %.2f ms, cuBLAS (no epilogues) %.2f ms" % (tot_o / 1e3, tot_c / 1e3))


if __name__ == "__main__":
    main()
