"""Images/s of batched solves against solo solves at the reference geometry (random weights): grids 1x2, 2x2 and 2x3 at 384
(Li = 1152, 2304, 3456; 30 time points) and the SDEdit solve at 1024^2 (Li = 4096; 10 time points, strength 0.4, no shift), at
batch 1, 2, 4 and the largest batch whose engine and decoder workspaces fit in free memory (at most 8).  For every batch B, one batched solve of B
samples and B solo solves alternate in one process; medians of the repeats.  Also the VAE decode of the query row (or of the
SDEdit image) for B images in one call against B calls.  Device time per image from CUDA events; SM clock and power read before
and after.  Writes the results as JSON to --out (default: bench_batch.json in $VCB_REPORT_DIR, else the system's temporary
directory).

Usage: python tools/bench_batch.py [--repeats N] [--shapes 1x2 2x2 2x3 sdedit] [--steps-scale S] [--max-batch B] [--out FILE]
(--steps-scale < 1 shortens every solve to that share of its time points; DESIGN.md §2g says which settings its table used)."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile

import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

from visualcloze_b200 import model as M, transport as T, vae as V  # noqa: E402

BF16 = torch.bfloat16
SHAPES = {  # name: (grid_h, grid_w, res, time points, do_shift, strength, query rows decoded (h, w) in pixels)
    "1x2": (1, 2, 384, 30, True, None, (384, 768)),
    "2x2": (2, 2, 384, 30, True, None, (384, 768)),
    "2x3": (2, 3, 384, 30, True, None, (384, 1152)),
    "sdedit": (1, 1, 1024, 10, False, 0.4, (1024, 1024)),
}


def gpu_state():
    q = "name,power.limit,clocks.sm,clocks.max.sm,power.draw"
    try:
        return subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True,
                              timeout=30).stdout.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError, IndexError):
        return "unavailable"


def inputs(gh, gw, res, B, seed):
    g = torch.Generator().manual_seed(seed)
    h, w = res // 16, gw * res // 16
    ids = []
    for j in range(gh):
        t = torch.zeros(h, w, 3)
        t[..., 0] = j + 1
        t[..., 1] += torch.arange(h)[:, None]
        t[..., 2] += torch.arange(w)[None, :]
        ids.append(t.reshape(-1, 3))
    img_ids = torch.cat(ids)[None].expand(B, -1, -1).contiguous()
    Li, Lt = img_ids.shape[1], 512
    x = torch.randn(B, Li, 64, generator=g).to(BF16)
    cond = torch.randn(B, Li, 320, generator=g).to(BF16)
    kw = dict(txt=(0.1 * torch.randn(B, Lt, 4096, generator=g)).to(BF16), txt_ids=torch.zeros(B, Lt, 3),
              txt_mask=torch.ones(B, Lt, dtype=torch.int32), y=torch.randn(B, 768, generator=g).to(BF16), img_ids=img_ids,
              img_mask=torch.ones(B, Li, dtype=torch.int32), cond=cond, guidance=torch.full((B,), 30.0, dtype=BF16))
    return x.cuda(), {k: v.cuda() for k, v in kw.items()}, Li


def timed(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--shapes", nargs="*", default=list(SHAPES))
    ap.add_argument("--steps-scale", type=float, default=1.0)
    ap.add_argument("--max-batch", type=int, default=8)
    ap.add_argument("--out", default=os.path.join(os.environ.get("VCB_REPORT_DIR") or tempfile.gettempdir(), "bench_batch.json"))
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_batch.py needs an H100: the hot path has no CPU fallback")
    out = {"gpu_before": gpu_state(), "repeats": args.repeats, "steps_scale": args.steps_scale, "shapes": {}}
    with torch.device("cuda"):
        model = M.FluxLoraWrapper(lora_rank=256, params=M.flux_dev_fill_params())
    model.init_synthetic(0)
    dec = V.AutoEncoderDecoder(device="cuda").init_synthetic(0)
    for name in args.shapes:
        gh, gw, res, steps, shift, strength, (qh, qw) = SHAPES[name]
        steps = max(2, round(steps * args.steps_scale))
        fn = T.Sampler(T.create_transport("Linear", "velocity", do_shift=True)).sample_ode(
            sampling_method="euler", num_steps=steps, atol=1e-6, rtol=1e-3, reverse=False, do_shift=shift,
            time_shifting_factor=1 if shift else 1.0, strength=strength)
        Li = gh * gw * (res // 16) ** 2
        eng = model.engine()
        free = torch.cuda.mem_get_info()[0] + (eng._ws.numel() if eng._ws is not None else 0) - (6 << 30)
        free += dec._ws.numel() if dec._ws is not None else 0
        bmax = max(b for b in range(1, args.max_batch + 1) if eng.lib.vcb_flux_workspace_bytes(eng._h, b, Li, 512, steps - 1)
                   + eng.lib.vcb_vae_workspace_bytes(dec._engine(), b, qh // 16, qw // 16) <= free)
        rows = {}
        for B in sorted({1, 2, 4, bmax}):
            if B > bmax:
                continue
            xb, kwb, _ = inputs(gh, gw, res, B, seed=B)
            solo = [({k: v[b:b + 1] for k, v in kwb.items()}, xb[b:b + 1]) for b in range(B)]
            tok = torch.randn(B, qh * qw // 256, 64, device="cuda").to(BF16)
            fn(xb, model.forward, kwb)                                   # warm-up of both shapes
            fn(solo[0][1], model.forward, solo[0][0])
            dec.decode_packed(tok, qh // 16, qw // 16)
            dec.decode_packed(tok[:1], qh // 16, qw // 16)
            t_b, t_s, d_b, d_s = [], [], [], []
            for _ in range(args.repeats):
                t_b.append(timed(lambda: fn(xb, model.forward, kwb)))
                t_s.append(timed(lambda: [fn(x1, model.forward, k1) for k1, x1 in solo]))
                d_b.append(timed(lambda: dec.decode_packed(tok, qh // 16, qw // 16)))
                d_s.append(timed(lambda: [dec.decode_packed(tok[b:b + 1], qh // 16, qw // 16) for b in range(B)]))
            mb, ms, vb, vs = (statistics.median(v) for v in (t_b, t_s, d_b, d_s))
            rows[B] = {"solve_ms_per_image_batched": mb / B, "solve_ms_per_image_solo": ms / B,
                       "vae_ms_per_image_batched": vb / B, "vae_ms_per_image_solo": vs / B,
                       "images_per_s_batched": 1000.0 * B / (mb + vb), "images_per_s_solo": 1000.0 * B / (ms + vs),
                       "solve_speedup": ms / mb, "spread_batched_ms": [min(t_b), max(t_b)], "spread_solo_ms": [min(t_s), max(t_s)]}
            print(f"{name} Li={Li} B={B}: solve {mb / B:.1f} vs {ms / B:.1f} ms/image (x{ms / mb:.3f}), VAE {vb / B:.1f} vs "
                  f"{vs / B:.1f} ms/image", flush=True)
            del xb, kwb, solo, tok
            torch.cuda.empty_cache()
        out["shapes"][name] = {"Li": Li, "time_points": steps, "largest_batch": bmax, "batches": rows}
    out["gpu_after"] = gpu_state()
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(out, f, indent=1)
    print(json.dumps({"gpu_before": out["gpu_before"], "gpu_after": out["gpu_after"]}))


if __name__ == "__main__":
    main()
