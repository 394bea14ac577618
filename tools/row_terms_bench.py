"""What row terms (DESIGN 6r) cost on the Elevation and Visual steps, arms alternating within one run:

(a) Elevation, one env step in a CUDA graph of T device-counter ``wl_step`` calls (step kernel + ray-cast kernel), N envs:
    the built-in row, row terms that restate it (no noise: the row kernel's clips and scales only), uniform noise on all
    689 columns, Gaussian noise on all 689 columns; CUDA events over the replays;
(b) Elevation, one whole training iteration of the fused runner (rollout of T steps, episode statistics, GAE, PPO update),
    ``FusedOnPolicyRunner.learn(1)`` timed with a device synchronise, with and without uniform noise on the height map;
(c) Visual, the graph of (a) at 512 envs (camera on): the built-in row against Gaussian / uniform noise on the 8 tail floats.

    python tools/row_terms_bench.py [--envs 4096] [--steps 128] [--rounds 3] --out results.json

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


def events_ms(fn, reps: int) -> float:
    fn(); torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def elev_terms(noise):
    from wheeledlab_b200 import row_terms
    return [(fn, noise, cl, sc) for fn, _, cl, sc in row_terms.registered("elevation", 10.0)]


def vis_terms(noise):
    from wheeledlab_b200 import row_terms
    return [(fn, noise, cl, sc) for fn, _, cl, sc in row_terms.registered("visual")]


def make_sim(spec, terms=None):
    import wheeledlab_b200 as wl
    spec.cfg.enable_corruption = 1
    sim = wl.WheeledSim(spec, DEV)
    if terms:
        sim.set_row_terms(terms)
    sim.startup(); sim.reset(None, 0)
    return sim


def step_graph(sim, T):
    """A CUDA graph of T device-counter steps; returns its replay."""
    from wheeledlab_b200.sim import WheeledSim
    n = sim.num_envs
    act = sim.synth_actions(0)
    out = (torch.empty((n, sim.obs_dim), device=DEV), torch.empty(n, device=DEV), torch.empty(n, dtype=torch.uint8, device=DEV),
           torch.empty(n, dtype=torch.uint8, device=DEV))
    sim.set_step_counter(0)
    g, s = torch.cuda.CUDAGraph(), torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s), torch.cuda.graph(g, stream=s):
        for k in range(T):
            sim.step(act, WheeledSim.device_counter_plus(k), out=out)
        sim.advance_counter(T)
    torch.cuda.current_stream().wait_stream(s)
    sim.set_step_counter(0)
    return lambda keep=(sim, act, out): g.replay()


def alternate(arms: dict, rounds: int, reps: int, per: int) -> dict:
    runs = {k: [] for k in arms}
    for _ in range(rounds):
        for k, f in arms.items():
            runs[k].append(events_ms(f, reps) * 1e3 / per)
    return {k: {"runs": v, "median": statistics.median(v)} for k, v in runs.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=128)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("row_terms_bench needs a CUDA device: nothing is measured without one")
    import wheeledlab_b200 as wl
    N, T = a.envs, a.steps
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    res = {"gpu": smi, "envs": N, "steps": T, "rounds": a.rounds}

    # (a) Elevation steps
    arms = {"builtin": None, "identity": elev_terms(None), "uniform_689": elev_terms(("uniform", -0.1, 0.1)),
            "gaussian_689": elev_terms(("gaussian", 0.0, 0.1))}
    arms = {k: step_graph(make_sim(wl.elevation_task(num_envs=N, seed=3), v), T) for k, v in arms.items()}
    res["elevation_graph_step_us"] = alternate(arms, a.rounds, 10, T)
    del arms

    # (b) Elevation runner iterations
    from wheeledlab_b200.env import ManagerBasedRLEnv
    from wheeledlab_b200.learner import FusedOnPolicyRunner
    from wheeledlab_b200.runs import agent_cfg
    runners = {}
    for name, noise in (("builtin", None), ("map_uniform", ("uniform", -0.1, 0.1))):
        spec = wl.elevation_task(num_envs=N, seed=3)
        spec.cfg.enable_corruption = 1
        env = ManagerBasedRLEnv(spec, device=DEV)
        if noise:
            t = elev_terms(None)
            t[5] = (t[5][0], noise, t[5][2], t[5][3])
            env.set_row_terms([(fn, fn, {"noise": nz, "clip": cl, "scale": sc}) for fn, nz, cl, sc in t])
        torch.manual_seed(0)
        r = FusedOnPolicyRunner(env, agent_cfg("relu", steps=T), device=DEV)
        r.learn(1)
        runners[name] = r
    it_ms = {k: [] for k in runners}
    for _ in range(a.rounds):
        for k, r in runners.items():
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(); r.learn(3); e1.record(); torch.cuda.synchronize()
            it_ms[k].append(e0.elapsed_time(e1) / 3)
    res["elevation_runner_iteration_ms"] = {k: {"runs": v, "median": statistics.median(v)} for k, v in it_ms.items()}
    del runners

    # (c) Visual steps
    arms = {"builtin": None, "uniform_8": vis_terms(("uniform", -0.1, 0.1)), "gaussian_8": vis_terms(("gaussian", 0.0, 0.1))}
    arms = {k: step_graph(make_sim(wl.visual_task(num_envs=512, seed=3, camera="aug"), v), T) for k, v in arms.items()}
    res["visual512_graph_step_us"] = alternate(arms, a.rounds, 10, T)
    line = json.dumps(res)
    print(line)
    if a.out:
        Path(a.out).parent.mkdir(parents=True, exist_ok=True)
        with open(a.out, "a") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
