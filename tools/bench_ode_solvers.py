"""Fixed-grid ODE solvers at cfg B (bench.make_inputs("B"): full FLUX.1-Fill geometry, LoRA r = 256 merged, synthetic weights) at
an equal budget of model evaluations: euler with 30 time points (29 evaluations), midpoint with 15 (28) and rk4 with 8 (28), in one
process, alternating, each warmed up first.  Prints one JSON object with, per solver:

  * per-image device time of the solve through the public sampler (CUDA events around it, median over the repeats), split into
    vcb_flux_prepare for that many evaluations (timed on its own), the stage kernels (their summed device time from a
    torch.profiler run of one solve, kept apart from the timed runs) and the evaluations (the rest);
  * the final latent's rel-L2 distance to a fine solution (rk4 with 31 time points, 120 evaluations) from the same noise.

The weights are random, so the distances say how fast each order converges on this velocity field and what it costs, not which
solver gives better images with trained weights.  The card name, power limit and SM clocks are read in the same call.
Usage: python tools/bench_ode_solvers.py [--repeats N]"""
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

SOLVERS = (("euler", 30), ("midpoint", 15), ("rk4", 8))
FINE = ("rk4", 31)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=3, help="timed images per solver (alternating)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_ode_solvers.py needs an H100: the hot path has no CPU fallback")
    import bench
    from bench_lora_modes import card
    from visualcloze_b200 import model as M, ops, transport as T
    dev = torch.device("cuda")
    with torch.device(dev):
        model = M.FluxLoraWrapper(lora_rank=256, params=M.flux_dev_fill_params())
    model.init_synthetic(0)
    x, kw, Li, Lt = bench.make_inputs("B", 1234)
    xg = x.to(dev)
    kwg = {k: v.to(dev) for k, v in kw.items()}
    sampler = T.Sampler(T.create_transport("Linear", "velocity", do_shift=True))

    def solve(method, n):
        fn = sampler.sample_ode(sampling_method=method, num_steps=n, atol=1e-6, rtol=1e-3, reverse=False, do_shift=True,
                                time_shifting_factor=1)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        lat = fn(xg, model.forward, kwg)[-1]
        b.record()
        torch.cuda.synchronize()
        return lat.float(), a.elapsed_time(b)

    res = {"card": card(), "workload": "B (cfg B: 2x3 grid at 384, L = %d + %d tokens), LoRA merged" % (Li, Lt)}
    fine = solve(*FINE)[0]
    res["fine"] = dict(method=FINE[0], points=FINE[1], evals=ops.ODE_STAGES[FINE[0]] * (FINE[1] - 1))
    times = {m: [] for m, _ in SOLVERS}
    finals = {}
    for m, n in SOLVERS:
        solve(m, n)                                                   # warm-up of this solver's shapes
    for _ in range(args.repeats):
        for m, n in SOLVERS:
            finals[m], ms = solve(m, n)
            times[m].append(ms)

    eng = model.engine()

    def prepare_ms(E):
        pkw = dict(txt=kwg["txt"], y=kwg["y"], img_ids=kwg["img_ids"], txt_ids=kwg["txt_ids"],
                   timesteps=torch.linspace(0.0, 0.97, E)[:, None], guidance=kwg["guidance"], txt_mask=kwg["txt_mask"],
                   img_mask=kwg["img_mask"], n_img_tokens=Li)
        out = []
        for _ in range(args.repeats + 1):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            eng.prepare(**pkw)
            b.record()
            torch.cuda.synchronize()
            out.append(a.elapsed_time(b))
        return statistics.median(out[1:])

    def stage_kernel_ms(method, n):
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            solve(method, n)
        evs = [e for e in prof.events() if "ode_stage_kernel" in e.name]
        return sum(e.device_time_total for e in evs) / 1e3, len(evs)

    for m, n in SOLVERS:
        E = ops.ODE_STAGES[m] * (n - 1)
        total = statistics.median(times[m])
        prep = prepare_ms(E)
        st_ms, st_n = stage_kernel_ms(m, n)
        res[m] = dict(points=n, evals=E, ms_per_image=total, ms_per_image_all=times[m], prepare_ms=prep, stage_kernels_ms=st_ms,
                      stage_kernel_launches=st_n, evaluations_ms=total - prep - st_ms, ms_per_evaluation=(total - prep - st_ms) / E,
                      final_vs_fine=float((finals[m] - fine).norm() / fine.norm()))
    res["card_after"] = card()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
