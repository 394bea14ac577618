"""Host time per eager wl_step: a bound step (sim.bind_step), 4096-env Drift, two env sets round-robin so that every step
after the first runs chained, 4000 steps per window with no synchronise inside it, six windows after one warm-up.  Prints
one JSON line: microseconds per step of each window, their median and each handle's chained-step count.

    python tools/step_host_cost.py"""
import json
import statistics
import sys
import time
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import torch
import wheeledlab_b200 as wl
dev = "cuda:0"
sims = [wl.WheeledSim(wl.make_task("drift", num_envs=4096, seed=s), dev) for s in (1, 2)]
for s in sims:
    s.startup(); s.reset(None, 0)
acts = torch.stack([sims[0].synth_actions(t) for t in range(8)])
outs = [(torch.empty((4096, 14), device=dev), torch.empty(4096, device=dev), torch.empty(4096, dtype=torch.uint8, device=dev),
         torch.empty(4096, dtype=torch.uint8, device=dev)) for _ in sims]
fns = [s.bind_step(acts[i], outs[i]) for i, s in enumerate(sims)]
tc = [0, 0]
res = []
for rep in range(7):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for k in range(4000):
        m = k & 1
        fns[m](tc[m]); tc[m] += 1
    t1 = time.perf_counter()
    torch.cuda.synchronize()
    res.append((t1 - t0) / 4000 * 1e6)
print(json.dumps({"host_us_per_step": res[1:], "median": statistics.median(res[1:]), "chained": [s.chained_step_count if hasattr(s, "chained_step_count") else None for s in sims]}))
