"""Time the full-size FLUX-DiT denoise loop (cfg B of SURVEY.md section 8) on one H100; dev tool, not the bench."""
import os
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from visualcloze_b200 import _lib, model as M, transport as T  # noqa: E402

steps = int(sys.argv[1]) if len(sys.argv) > 1 else 30
rows = int(sys.argv[2]) if len(sys.argv) > 2 else 2
cols = int(sys.argv[3]) if len(sys.argv) > 3 else 3
res = 384
t0 = time.time()
with torch.device("cuda"):
    model = M.FluxLoraWrapper(lora_rank=256, params=M.flux_dev_fill_params())
model.init_synthetic(0)
torch.cuda.synchronize()
print(f"init {time.time() - t0:.1f}s, params {sum(p.numel() for p in model.parameters()) / 1e9:.2f} B", flush=True)
t0 = time.time()
eng = model.engine()
torch.cuda.synchronize()
print(f"pack {time.time() - t0:.1f}s, mem {torch.cuda.memory_allocated() / 2**30:.1f} GiB", flush=True)

h, w = res // 16, cols * res // 16
ids = []
for j in range(rows):
    t = torch.zeros(h, w, 3)
    t[..., 0] = j + 1
    t[..., 1] += torch.arange(h)[:, None]
    t[..., 2] += torch.arange(w)[None, :]
    ids.append(t.reshape(-1, 3))
ids = torch.cat(ids)[None].cuda()
Li, Lt = ids.shape[1], 512
g = torch.Generator().manual_seed(1234)
x = torch.randn(1, Li, 64, generator=g).to(torch.bfloat16).cuda()
cond = torch.randn(1, Li, 320, generator=g).to(torch.bfloat16).cuda()
kw = dict(txt=(0.1 * torch.randn(1, Lt, 4096, generator=g)).to(torch.bfloat16).cuda(), txt_ids=torch.zeros(1, Lt, 3).cuda(),
          txt_mask=torch.ones(1, Lt, dtype=torch.int32).cuda(), y=torch.randn(1, 768, generator=g).to(torch.bfloat16).cuda(),
          img_ids=ids, img_mask=torch.ones(1, Li, dtype=torch.int32).cuda(), cond=cond,
          guidance=torch.full((1,), 30.0, dtype=torch.bfloat16).cuda())
fn = T.Sampler(T.create_transport("Linear", "velocity", do_shift=True)).sample_ode(
    sampling_method="euler", num_steps=steps, atol=1e-6, rtol=1e-3, reverse=False, do_shift=True, time_shifting_factor=1)
for it in range(3):
    _lib.lib().vcb_reset_launch_count()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0 = time.time()
    e0.record()
    traj = fn(x, model.forward, kw)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1)
    print(f"iter {it}: {ms:.1f} ms total, {ms / (steps - 1):.2f} ms/NFE, wall {time.time() - t0:.3f}s, launches "
          f"{_lib.lib().vcb_launch_count()}, Li={Li}, finite={bool(torch.isfinite(traj[-1].float()).all())}, "
          f"absmean={traj[-1].float().abs().mean().item():.3f}", flush=True)
