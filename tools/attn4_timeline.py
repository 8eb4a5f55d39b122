"""Where does the persistent attention kernel's time go?  Per-CTA globaltimer stamps (VCB_ATTN4_TIMELINE=1) of one launch:
start, end of every segment.  Run twice: default (split tail) and VCB_ATTN4_NOSPLIT=1 (whole units).  Prints per-launch time of
the per-tile grid / the persistent schedule and, for the latter, the distribution of per-CTA phase durations."""
import ctypes as C
import math
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from visualcloze_b200 import _lib, ops  # noqa: E402

BF16 = torch.bfloat16
L = int(sys.argv[1]) if len(sys.argv) > 1 else 3968
heads = int(sys.argv[2]) if len(sys.argv) > 2 else 24
H = heads * 128
g = torch.Generator(device="cuda").manual_seed(0)
qkv = torch.randn(L, 3, heads, 128, generator=g, device="cuda")
for i, a in ((0, 1.2), (1, 1.1)):
    qkv[:, i] = a * qkv[:, i] / qkv[:, i].pow(2).mean(-1, keepdim=True).sqrt()
qkv = qkv.reshape(L, 3 * H).to(BF16)
out = torch.empty(L, H, dtype=BF16, device="cuda")
bound = 1.2 * 1.1 * math.sqrt(128.0) * math.log2(math.e) * 1.03
flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device="cuda")


def t(sched):
    f = lambda: ops.attention(qkv, 1, L, heads, out, q_col=0, k_col=H, v_col=2 * H, score_bound_log2=bound, schedule=sched)
    for _ in range(3):
        f()
    ts = []
    for _ in range(9):
        flush.zero_()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); f(); b.record(); torch.cuda.synchronize()
        ts.append(a.elapsed_time(b) * 1e3)
    return sorted(ts)[4]


print(f"L={L} heads={heads} split={'no' if os.environ.get('VCB_ATTN4_NOSPLIT') else 'yes'}: per-pair {t(1):.1f} us, persistent {t(2):.1f} us")
S = 66
buf = (C.c_ulonglong * (160 * S))()
flush.zero_()
ops.attention(qkv, 1, L, heads, out, q_col=0, k_col=H, v_col=2 * H, score_bound_log2=bound, schedule=2)
G = _lib.lib().vcb_debug_attn4_timeline(buf, 160 * S)
if G > 0:
    rows = [[buf[c * S + i] for i in range(S)] for c in range(G)]
    t0 = min(r[0] for r in rows if r[0])
    ends = [max(x for x in r if x) - t0 for r in rows]
    starts = [r[0] - t0 for r in rows]
    print(f"  grid {G}: CTA start spread {max(starts) / 1e3:.1f} us; CTA end min/median/max {min(ends) / 1e3:.1f} / {sorted(ends)[G // 2] / 1e3:.1f} / {max(ends) / 1e3:.1f} us")
    nseg = [sum(1 for x in r[1:] if x) for r in rows]
    print("  segments per CTA:", sorted(set(nseg)), " per-segment durations (us) of CTA 0, G/2, G-1:")
    for c in (0, G // 2, G - 1):
        st = [r for r in rows[c] if r]
        print(f"    cta {c}:", [round((st[i + 1] - st[i]) / 1e3, 1) for i in range(len(st) - 1)])
    # duration of the LAST segment and of the first tail segment across CTAs
    last = [(lambda st: (st[-1] - st[-2]) / 1e3)([x for x in r if x]) for r in rows if sum(1 for x in r if x) >= 2]
    print(f"  last-segment duration min/median/max: {min(last):.1f} / {sorted(last)[len(last) // 2]:.1f} / {max(last):.1f} us")
