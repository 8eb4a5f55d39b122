"""First-block cache at cfg B (bench.make_inputs("B"): full FLUX.1-Fill geometry, LoRA r = 256 merged, synthetic weights): the
cache off against several thresholds and a huge one that skips every evaluation after the first (the upper bound), all settings
in one process, alternating, each warmed up first.  Prints one JSON object with, per setting:

  * per-image device time of a 30-point Euler solve through the public sampler (vcb_flux_prepare + 29 evaluations + the Euler
    updates), CUDA events around the solve, median over the repeats;
  * evaluations computed / skipped;
  * the final latent's rel-L2 distance to the uncached solve.

The thresholds default to quartiles of the per-step diffs of a run that never skips (these weights are random: the numbers say
what a skip costs, not which threshold suits a trained model).  From the off and upper-bound settings, with vcb_flux_prepare timed
on its own, it derives the time of one computed and one skipped evaluation and sets the skipped one against its FLOP floor
(img_in + 1 of the 57 blocks + the final layer, over a whole evaluation).  The card name, power limit and SM clocks are read in
the same call.  Usage: python tools/bench_first_block_cache.py [--repeats N] [--thresholds T ...]"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys

import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "tools"))

STEPS = 30
UPPER = 1e30


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=3, help="timed images per setting (alternating)")
    ap.add_argument("--thresholds", type=float, nargs="*", default=None, help="default: quartiles of the observed diffs")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_first_block_cache.py needs an H100: the hot path has no CPU fallback")
    import bench
    from bench_lora_modes import card
    from visualcloze_b200 import model as M, transport as T
    dev = torch.device("cuda")
    with torch.device(dev):
        model = M.FluxLoraWrapper(lora_rank=256, params=M.flux_dev_fill_params())
    model.init_synthetic(0)
    x, kw, Li, Lt = bench.make_inputs("B", 1234)
    xg = x.to(dev)
    kwg = {k: v.to(dev) for k, v in kw.items()}
    fn = T.Sampler(T.create_transport("Linear", "velocity", do_shift=True)).sample_ode(
        sampling_method="euler", num_steps=STEPS, atol=1e-6, rtol=1e-3, reverse=False, do_shift=True, time_shifting_factor=1)

    def solve(threshold, diffs=None):
        model.enable_first_block_cache(threshold)
        eng = model.engine()
        if diffs is not None:
            fwd = eng.forward

            def rec(*a, **k):
                out = fwd(*a, **k)
                diffs.append(eng.cache_stats()["last_diff"])
                return out
            eng.forward = rec
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        lat = fn(xg, model.forward, kwg)[-1]
        b.record()
        torch.cuda.synchronize()
        eng.__dict__.pop("forward", None)
        return lat.float(), a.elapsed_time(b), eng.cache_stats()

    res = {"card": card(), "workload": "B (cfg B: 2x3 grid at 384, L = %d + %d tokens)" % (Li, Lt), "evals": STEPS - 1}
    solve(None)                                                    # warm-up: module load, workspace, stream-K scratch
    diffs = []
    solve(1e-30, diffs)                                            # cache on, never skipping: the per-step diffs
    ds = sorted(d for d in diffs[1:])
    res["observed_diffs"] = diffs[1:]
    thresholds = args.thresholds if args.thresholds else [ds[len(ds) // 4], ds[len(ds) // 2], ds[3 * len(ds) // 4]]
    settings = [None] + thresholds + [UPPER]
    name = lambda t: "off" if t is None else ("upper_bound" if t == UPPER else f"threshold_{t:.4g}")
    base = solve(None)[0]
    times = {name(t): [] for t in settings}
    out = {}
    for t in settings:
        solve(t)                                                   # warm-up of this setting
    for _ in range(args.repeats):
        for t in settings:
            lat, ms, st = solve(t)
            times[name(t)].append(ms)
            out[name(t)] = dict(threshold=t, computed=st["computed"], skipped=st["skipped"], final_vs_uncached=
                                float((lat - base).norm() / base.norm()))
    for k, v in out.items():
        v.update(ms_per_image=statistics.median(times[k]), ms_per_image_all=times[k])
        res[k] = v
    # vcb_flux_prepare alone, to split the solve into prepare + evaluations
    model.enable_first_block_cache(None)
    eng = model.engine()
    pkw = dict(txt=kwg["txt"], y=kwg["y"], img_ids=kwg["img_ids"], txt_ids=kwg["txt_ids"],
               timesteps=torch.linspace(0.0, 0.97, STEPS - 1)[:, None], guidance=kwg["guidance"], txt_mask=kwg["txt_mask"],
               img_mask=kwg["img_mask"], n_img_tokens=Li)
    prep = []
    for _ in range(args.repeats + 1):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        eng.prepare(**pkw)
        b.record()
        torch.cuda.synchronize()
        prep.append(a.elapsed_time(b))
    prep_ms = statistics.median(prep[1:])
    n = STEPS - 1
    computed_ms = (res["off"]["ms_per_image"] - prep_ms) / n
    skipped_ms = (res["upper_bound"]["ms_per_image"] - prep_ms - computed_ms) / (n - 1)
    H, L = 3072, Li + Lt
    per_eval = 2 * Li * 384 * H + 57 * 24 * L * H * H + 2 * Li * H * 64 + 57 * 4 * L * L * H
    floor = 2 * Li * 384 * H + 24 * L * H * H + 4 * L * L * H + 2 * Li * H * 64
    res["split"] = dict(prepare_ms=prep_ms, computed_eval_ms=computed_ms, skipped_eval_ms=skipped_ms,
                        skipped_over_computed=skipped_ms / computed_ms, flop_floor_skipped_over_computed=floor / per_eval)
    res["card_after"] = card()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
