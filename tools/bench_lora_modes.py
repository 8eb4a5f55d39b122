"""Merged vs unmerged LoRA at cfg B (bench.make_inputs("B"): full FLUX.1-Fill geometry, r = 256, synthetic weights), both
modes in one process, alternating, each warmed up first.  Prints one JSON object with, per mode:

  * per-image device time of the 29 model evaluations of a 30-point trajectory (vcb_flux_prepare + 29 vcb_flux_forward;
    the Euler updates, equal in both modes, are left out), median over the repeats, host clock around a device synchronise;
  * the GEMM share of one image from the per-launch records of vcb_profile_end_ex, split into main GEMMs and LoRA
    down-projections (records with N == 256, the rank; the final layer's rank-64 down-projection, one small launch per
    evaluation, is booked with the main GEMMs);
  * torch.cuda.memory_allocated() added by building the engine;
  * latency of set_lora_scale + the next engine(), and of an adapter swap by load_state_dict(..., strict=False, assign=True) +
    engine() (two full-size adapters resident).

The card name, power limit and SM clocks are read in the same call.  Usage: python tools/bench_lora_modes.py [--repeats N]"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

RANK = 256
EVALS = 29


def card() -> dict:
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader,nounits", "-i", str(torch.cuda.current_device())],
                           capture_output=True, text=True, timeout=30)
        name, pl, sm, smax = [s.strip() for s in r.stdout.strip().splitlines()[0].split(",")]
        return {"name": name, "power_limit_w": float(pl), "sm_clock_mhz": float(sm), "sm_clock_max_mhz": float(smax)}
    except Exception as e:                                    # the measurement itself does not depend on it
        return {"name": torch.cuda.get_device_name(), "nvidia_smi": f"unavailable ({e})"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5, help="timed images per mode (alternating)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_lora_modes.py needs an H100: the hot path has no CPU fallback")
    import bench
    from visualcloze_b200 import _lib, model as M
    from visualcloze_b200.engine import FluxEngine
    lib = _lib.lib()
    dev = torch.device("cuda")
    with torch.device(dev):
        model = M.FluxLoraWrapper(lora_rank=RANK, params=M.flux_dev_fill_params())
    model.init_synthetic(0)
    x, kw, Li, Lt = bench.make_inputs("B", 1234)
    img = torch.cat((x, kw.pop("cond")), dim=-1).to(dev)
    ts = torch.linspace(0.0, 0.97, EVALS)[:, None]
    pkw = dict(txt=kw["txt"].to(dev), y=kw["y"].to(dev), img_ids=kw["img_ids"].to(dev), txt_ids=kw["txt_ids"].to(dev),
               timesteps=ts, guidance=kw["guidance"].to(dev), txt_mask=kw["txt_mask"].to(dev), img_mask=kw["img_mask"].to(dev),
               n_img_tokens=Li)

    def build(mode):
        torch.cuda.synchronize()
        before = torch.cuda.memory_allocated()
        eng = FluxEngine(model.params, dict(model.named_parameters()), model.lora_scale, lora_mode=mode)
        torch.cuda.synchronize()
        return eng, torch.cuda.memory_allocated() - before

    def image(eng):
        eng.prepare(**pkw)
        out = None
        for e in range(EVALS):
            out = eng.forward(e, img, out)
        return out

    res = {"card": card(), "workload": "B (cfg B: 2x3 grid at 384, L = %d + %d tokens)" % (Li, Lt), "rank": RANK, "evals": EVALS}
    engines, modes = {}, ("merged", "unmerged")
    for mode in modes:
        engines[mode], added = build(mode)
        res[mode] = {"engine_build_bytes": added}
        image(engines[mode])                                   # warm-up: module load, workspace, stream-K scratch
    times = {m: [] for m in modes}
    for _ in range(args.repeats):
        for mode in modes:
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            image(engines[mode])
            torch.cuda.synchronize()
            times[mode].append(time.perf_counter() - t0)
    for mode in modes:
        lib.vcb_profile_begin()
        image(engines[mode])
        cats, recs = _lib.profile_end(max_records=40000)
        gemm = [r for r in recs if r.category == 0]
        down = sum(r.ms for r in gemm if r.info[1] == RANK)
        res[mode].update(ms_per_image=1000 * statistics.median(times[mode]), ms_per_image_all=[1000 * t for t in times[mode]],
                         profiled_gemm_ms=sum(r.ms for r in gemm), profiled_gemm_main_ms=sum(r.ms for r in gemm) - down,
                         profiled_down_projection_ms=down, profiled_attention_ms=cats["attention"][0],
                         profiled_total_ms=sum(v[0] for v in cats.values()), gemm_launches=len(gemm))
    res["unmerged_over_merged"] = res["unmerged"]["ms_per_image"] / res["merged"]["ms_per_image"]
    res["down_projection_share_of_unmerged_gemm"] = res["unmerged"]["profiled_down_projection_ms"] / res["unmerged"]["profiled_gemm_ms"]
    engines.clear()

    # ---- rebuild latencies through the public model API ----
    names = [n for n, _ in model.named_parameters() if ".lora_" in n]
    adapters = []
    for seed in (1, 2):
        g = torch.Generator(device=dev).manual_seed(seed)
        adapters.append({n: 0.02 * torch.randn(model.get_parameter(n).shape, generator=g, device=dev, dtype=torch.bfloat16) for n in names})
    for mode in modes:
        model.set_lora_mode(mode)
        model.set_lora_scale(1.0)
        model.engine()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        model.set_lora_scale(0.8)
        model.engine()
        torch.cuda.synchronize()
        res[mode]["set_lora_scale_s"] = time.perf_counter() - t0
        swaps = []
        for ad in adapters:
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            model.load_state_dict(ad, strict=False, assign=True)
            model.engine()
            torch.cuda.synchronize()
            swaps.append(time.perf_counter() - t0)
        res[mode]["adapter_swap_s"] = swaps
        model._engine = None
        torch.cuda.empty_cache()
    res["card_after"] = card()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
