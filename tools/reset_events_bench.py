"""What the reset-mode DR events (DESIGN 6n) cost: each case with mask 0 (start-up DR only) and with every event the task has
in reset mode, the two arms alternating within one run, CUDA events over graph replays:

(a) Drift N: a CUDA graph of T ``wl_act_step`` launches (FusedPolicyRollout), time per step;
(b) Drift N: one whole runner iteration graph (PPOIteration: rollout, episode statistics, bootstrap, GAE, PPO update);
(c) HOUND-4WD 2N: a CUDA graph of T ``wl_step`` launches on the device counter, time per step.

    python tools/reset_events_bench.py [--envs 4096] [--steps 128] [--rounds 3] --out results.jsonl

The card's name and power limit are read in the same run and written beside the figures.
"""
from __future__ import annotations

import argparse
import json
import statistics
import subprocess
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
DEV = "cuda:0"
D = 14
EVENTS = {"mask0": {}, "all": {"material": True, "actuator_gains": True, "base_mass": True}}


def events_ms(fn, reps: int) -> float:
    fn(); torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def make_sim(task, n, events):
    import wheeledlab_b200 as wl
    sim = wl.WheeledSim(wl.make_task(task, num_envs=n, seed=3), DEV)
    sim.set_reset_events(**events)
    sim.startup(); sim.reset(None, 0)
    return sim


def blob():
    from wheeledlab_b200.policy import pack_actor_critic
    torch.manual_seed(0)
    mk = lambda nin, out: torch.nn.Sequential(torch.nn.Linear(nin, 64), torch.nn.ELU(), torch.nn.Linear(64, 64), torch.nn.ELU(),
                                              torch.nn.Linear(64, out))
    return pack_actor_critic(mk(D, 2), mk(D, 1), torch.ones(2), D, DEV)


def step_graph(sim, T):
    """T x wl_step on the device counter, then wl_advance_counter(T): one replayable graph."""
    n = sim.num_envs
    act = sim.synth_actions(0)
    out = (torch.empty(n, sim.obs_dim, device=DEV), torch.empty(n, device=DEV), torch.empty(n, dtype=torch.uint8, device=DEV),
           torch.empty(n, dtype=torch.uint8, device=DEV))
    sim.set_step_counter(1)
    g, cs = torch.cuda.CUDAGraph(), torch.cuda.Stream()
    cs.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(cs):
        sim.step(act, sim.device_counter_plus(0), out=out)              # warm-up (module load) outside the capture
        sim.advance_counter(1)
        with torch.cuda.graph(g, stream=cs):
            for k in range(T):
                sim.step(act, sim.device_counter_plus(k), out=out)
            sim.advance_counter(T)
    torch.cuda.current_stream().wait_stream(cs)
    keep = (sim, act, out, g)              # the graph reads the handle, its state buffer and these tensors at every replay

    def replay(_keep=keep):
        g.replay()
    return replay


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=128)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("reset_events_bench needs a CUDA device: nothing is measured without one")
    from wheeledlab_b200.learner import PPOConfig, PPOIteration
    from wheeledlab_b200.policy import FusedPolicyRollout
    N, T = a.envs, a.steps
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    res = {"gpu": smi, "envs": N, "steps": T, "rounds": a.rounds}
    cases = {}
    for arm, ev in EVENTS.items():
        cases[f"drift_act_step_{arm}"] = (FusedPolicyRollout(make_sim("drift", N, ev), blob(), T).capture(0).run, 20, T)
        it = PPOIteration(make_sim("drift", N, ev), blob(), PPOConfig(), T, episode_stats=True).start(0, capture=True)
        cases[f"drift_iteration_{arm}"] = (it.run, 10, 1)
        cases[f"hound4wd_{2 * N}_step_{arm}"] = (step_graph(make_sim("hound_4wd", 2 * N, ev), T), 20, T)
    runs = {k: [] for k in cases}
    for _ in range(a.rounds):
        for k, (fn, reps, per) in cases.items():
            runs[k].append(events_ms(fn, reps) * (1e3 / per if per > 1 else 1.0))
    res["us_per_step"] = {k: {"runs": v, "median": statistics.median(v)} for k, v in runs.items() if cases[k][2] > 1}
    res["ms_per_iteration"] = {k: {"runs": v, "median": statistics.median(v)} for k, v in runs.items() if cases[k][2] == 1}
    line = json.dumps(res)
    print(line)
    if a.out:
        Path(a.out).parent.mkdir(parents=True, exist_ok=True)
        with open(a.out, "a") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
