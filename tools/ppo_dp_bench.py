"""Cost of the data-parallel PPO update on one GPU (DESIGN 6j): wl_ppo_update_dp with one rank against wl_ppo_update /
wl_ppo_update_wide (the publish, DP-reduce and exchange-slot traffic it adds), and a whole captured training iteration
in the single-rank form against the one-process data-parallel form (R = 1, and R = 2 ranks of half the envs).

Drift (obs_dim 14, ELU) and Elevation (689, ReLU) at 4096 envs x 128 steps, the reference agent cfg (5 epochs x 4
mini-batches); the update timings alternate the two paths over three runs; CUDA events around `--reps` calls after two
warm-up calls.  One JSON line per measurement, also written to --out.

    python tools/ppo_dp_bench.py --out results/h100/ppo_dp/bench.jsonl
"""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
sys.path.insert(0, str(Path(__file__).resolve().parent.parent / "tests"))
DEV = "cuda:0"


def _time(fn, reps):
    for _ in range(2):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def update_rows(name, D, activation, reps, runs):
    from test_ppo_dp_gpu import _synthetic
    from wheeledlab_b200.learner import FusedPPO, PPOConfig, PPOExchange, update_local_ranks
    cfg = PPOConfig()
    blob, [(slab, ret, adv, perm)] = _synthetic(D, activation, 1, 4096 * 128, seed=1)
    single = FusedPPO(blob.clone(), D, cfg, activation)
    dp = FusedPPO(blob.clone(), D, cfg, activation, exchange=PPOExchange.local(1, D, DEV)[0])
    out = []
    for run in range(runs):
        for path, fn in (("single", lambda: single.update(slab, ret, adv, perm)),
                         ("dp_r1", lambda: update_local_ranks([dp], [(slab, ret, adv, perm)]))):
            out.append({"what": "update", "task": name, "obs_dim": D, "path": path, "run": run + 1, "rows": 4096 * 128,
                        "ms_per_update": _time(fn, reps)})
    return out


def iteration_rows(reps):
    import wheeledlab_b200 as wl
    from test_ppo_dp_gpu import _nets
    from wheeledlab_b200.learner import LocalRanksIteration, PPOConfig, PPOExchange, PPOIteration
    from wheeledlab_b200.policy import pack_actor_critic
    actor, critic, _ = _nets(14, "elu", 3)
    blob = pack_actor_critic(actor, critic, torch.ones(2, device=DEV), 14, DEV)
    T, total = 128, 4096

    def sim(n, r):
        s = wl.WheeledSim(wl.drift_task(num_envs=n, seed=5, env_id_offset=r * n), DEV); s.startup(); s.reset(None, 0)
        return s

    def group(R):
        n = total // R
        return LocalRanksIteration([PPOIteration(sim(n, r), blob.clone(), PPOConfig(), T, episode_stats=True, exchange=ex)
                                    for r, ex in enumerate(PPOExchange.local(R, 14, DEV))]).start(0)

    forms = (("single", lambda: PPOIteration(sim(total, 0), blob.clone(), PPOConfig(), T, episode_stats=True).start(0)),
             ("dp_one_process_r1", lambda: group(1)), ("dp_one_process_r2", lambda: group(2)))
    out = []
    for form, mk in forms:
        it = mk()
        out.append({"what": "iteration_graph", "task": "drift", "form": form, "envs": total, "T": T,
                    "ms_per_iteration": _time(it.run, reps)})
        del it
        torch.cuda.synchronize()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()[0]
    rows = [{"gpu": gpu, "torch": torch.__version__}]
    rows += update_rows("drift", 14, "elu", a.reps, a.runs)
    rows += update_rows("elevation", 689, "relu", a.reps, a.runs)
    rows += iteration_rows(a.reps)
    text = "\n".join(json.dumps(r) for r in rows)
    print(text)
    if a.out:
        Path(a.out).parent.mkdir(parents=True, exist_ok=True)
        Path(a.out).write_text(text + "\n")


if __name__ == "__main__":
    main()
