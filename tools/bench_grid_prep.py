"""Grid-cell preparation of ``VisualClozeModel.process_images``: host wall time, ending in a device synchronise, of turning the
caller's in-memory RGB images into the model input rows, on the Pillow path (``convert`` + ``_prepare_grid`` + ``image_transform``
+ ``torch.cat`` + upload, what the pipeline did before) and on the device path (``convert`` + ``_grid_rows``: one upload per image,
libvcb200's resampler and the store kernel), alternating in one process, median over the repeats, each workload warmed up first.

Workloads: 2x3 with one target (five inputs) and 3x4 with three targets
(nine inputs), of 4032x3024 and of 1024x1024 images, resolution 384.  The device path is split, in a separate instrumented run,
into the upload (host wall time of np.asarray + pinned staging + copy, synchronised per image) and the kernels (device time from
CUDA events around every libvcb200 launch, vcb_profile_end).  Random pixel content; no JPEG decode.  The card name, power limit
and SM clocks are read in the same call, and the host CPU model is printed beside the Pillow numbers.
Usage: python tools/bench_grid_prep.py [--repeats N]"""
from __future__ import annotations

import argparse
import json
import os
import platform
import statistics
import sys
import time

import numpy as np
import torch
from PIL import Image

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "tools"))

WORKLOADS = (("2x3, one target, five 4032x3024", 2, 3, 1, (4032, 3024)),
             ("3x4, three targets, nine 4032x3024", 3, 4, 3, (4032, 3024)),
             ("2x3, one target, five 1024x1024", 2, 3, 1, (1024, 1024)),
             ("3x4, three targets, nine 1024x1024", 3, 4, 3, (1024, 1024)))


def cpu_model() -> str:
    try:
        for line in open("/proc/cpuinfo"):
            if line.startswith("model name"):
                return line.split(":", 1)[1].strip()
    except OSError:
        pass
    return platform.processor() or "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5, help="timed runs per path and workload (alternating)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_grid_prep.py needs an H100: the device path has no CPU fallback")
    from bench_lora_modes import card
    from visualcloze_b200 import _lib, pipeline as P, resample
    dev = torch.device("cuda")
    rng = np.random.default_rng(0)
    res = {"card": card(), "host_cpu": cpu_model(), "torch_threads": torch.get_num_threads(), "resolution": 384, "workloads": []}

    for name, gh, gw, n_targets, (w, h) in WORKLOADS:
        pm = object.__new__(P.VisualClozeModel)
        pm.grid_h, pm.grid_w, pm.resolution, pm.device = gh, gw, 384, dev
        pool = [Image.fromarray(rng.integers(0, 256, (h, w, 3), dtype=np.uint8)) for _ in range(gh * gw - n_targets)]

        def grid():
            it = iter(pool)
            return [[None if (i == gh - 1 and j >= gw - n_targets) else next(it) for j in range(gw)] for i in range(gh)]

        def pillow():
            imgs = [[im.convert("RGB") if im is not None else None for im in row] for row in grid()]
            cells, _, _ = pm._prepare_grid(imgs)
            rows = [torch.cat([P.image_transform(c) for c in cells[i * gw:(i + 1) * gw]], dim=2).to(dev) for i in range(gh)]
            torch.cuda.synchronize()
            return rows

        def device():
            imgs = [[im.convert("RGB") if im is not None else None for im in row] for row in grid()]
            rows = pm._grid_rows(imgs)[0]
            torch.cuda.synchronize()
            return rows

        a, b = pillow(), device()                                   # warm-up: tables, allocator, pinned staging
        assert all(torch.equal(x, y) for x, y in zip(a, b)), f"{name}: device rows differ from the Pillow rows"
        times = {"pillow": [], "device": []}
        for _ in range(args.repeats):
            for tag, fn in (("pillow", pillow), ("device", device)):
                t0 = time.perf_counter()
                fn()
                times[tag].append((time.perf_counter() - t0) * 1e3)

        # instrumented run of the device path: upload (synchronised per image) and kernel device time
        upload = resample.upload
        up_ms = []

        def timed_upload(image, device_):
            t0 = time.perf_counter()
            t = upload(image, device_)
            torch.cuda.synchronize()
            up_ms.append((time.perf_counter() - t0) * 1e3)
            return t
        resample.upload = timed_upload
        try:
            _lib.check(_lib.lib().vcb_profile_begin(), "vcb_profile_begin")
            device()
            cats, _ = _lib.profile_end()
        finally:
            resample.upload = upload
        res["workloads"].append({
            "workload": name, "inputs": len(pool),
            "pillow_ms_median": statistics.median(times["pillow"]), "device_ms_median": statistics.median(times["device"]),
            "pillow_ms": [round(t, 2) for t in times["pillow"]], "device_ms": [round(t, 2) for t in times["device"]],
            "device_upload_ms": round(sum(up_ms), 3), "device_kernel_ms": round(cats["other"][0], 3),
            "device_kernel_launches": cats["other"][1],
            "speedup": statistics.median(times["pillow"]) / statistics.median(times["device"]),
        })
        print(json.dumps(res["workloads"][-1]), flush=True)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
