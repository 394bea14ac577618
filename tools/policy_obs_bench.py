"""What a policy observation table (DESIGN 6q) costs, Drift N x T, arms alternating within one run:

(a) ``wl_policy_observe`` alone, CUDA events over eager launches, at Dp = 11 (BlindObsCfg without root_pos_w) and Dp = 32
    (every noise kind, clips and scales), N = 4096 and 8192;
(b) one env step in a CUDA graph of T steps: ``wl_step`` alone against ``wl_step`` + ``wl_policy_observe`` (Dp = 11), both
    on device counters, CUDA events over the replays;
(c) ``wl_policy_observe`` alone in a CUDA graph of T launches (Dp = 11 and 32): the kernel without the host's launch cost;
(d) one whole training iteration graph (rollout, episode statistics, bootstrap, GAE, update; ``PPOIteration``): the fused
    symmetric network on the built-in row against the network on the Dp = 11 table (policy kernel, step, row per step).

    python tools/policy_obs_bench.py [--envs 4096] [--steps 128] [--rounds 3] --out results.json

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
NO_POS = [("root_euler_xyz", ("gaussian", 0.0, 0.1), None, None), ("base_lin_vel", ("gaussian", 0.0, 0.5), None, None),
          ("base_ang_vel", ("gaussian", 0.0, 0.4), None, None), ("last_action", None, (-1.0, 1.0), None)]
WIDE = [("projected_gravity", ("gaussian", 0.0, 0.05), None, None), ("base_ang_vel", ("gaussian", 0.0, 0.4), None, None),
        ("base_lin_vel", ("uniform", -0.5, 0.5), None, None), ("last_action", None, (-1.0, 1.0), None),
        ("joint_vel", ("gaussian", 0.1, 0.2), None, 0.01), ("joint_pos", ("uniform", 0.0, 0.1), (-0.3, 0.2), None),
        ("wheel_friction", ("gaussian", 0.0, 0.1), None, None), ("base_mass", ("uniform", -1.0, 1.0), None, 0.5),
        ("motor_damping", None, (-0.5, 0.5), (1.0, 2.0, 3.0, 4.0)), ("root_euler_xyz", ("gaussian", 0.0, 0.1), None, None),
        ("root_pos_w", None, None, None)]


def events_ms(fn, reps: int) -> float:
    fn(); torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def make_sim(n, table=None):
    import wheeledlab_b200 as wl
    sim = wl.WheeledSim(wl.drift_task(num_envs=n, seed=3), DEV); sim.startup(); sim.reset(None, 0)
    if table:
        sim.set_policy_terms(table)
    return sim


def step_graph(sim, T, observe: bool, step: bool = True):
    """A CUDA graph of T device-counter steps (and the table's row after each when `observe`, only the rows when not `step`);
    returns its replay."""
    from wheeledlab_b200.sim import WheeledSim
    n = sim.num_envs
    act = sim.synth_actions(0)
    out = (torch.empty((n, sim.obs_dim), device=DEV), torch.empty(n, device=DEV), torch.empty(n, dtype=torch.uint8, device=DEV),
           torch.empty(n, dtype=torch.uint8, device=DEV))
    pobs = torch.empty((T, n, max(1, sim.policy_obs_dim)), device=DEV)
    sim.set_step_counter(0)
    g, s = torch.cuda.CUDAGraph(), torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s), torch.cuda.graph(g, stream=s):
        for k in range(T):
            if step:
                sim.step(act, WheeledSim.device_counter_plus(k), out=out)
            if observe:
                sim.policy_observe(WheeledSim.device_counter_plus(k), out=pobs[k])
        sim.advance_counter(T)
    torch.cuda.current_stream().wait_stream(s)
    sim.set_step_counter(0)
    return lambda keep=(sim, act, out, pobs): g.replay()     # the graph writes these: they live as long as the replay


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=128)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("policy_obs_bench needs a CUDA device: nothing is measured without one")
    N, T = a.envs, a.steps
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    res = {"gpu": smi, "envs": N, "steps": T, "rounds": a.rounds}

    # (a) the kernel alone
    obs = {}
    for n in (N, 2 * N):
        for name, table in (("dp11", NO_POS), ("dp32", WIDE)):
            sim = make_sim(n, table)
            out = torch.empty((n, sim.policy_obs_dim), device=DEV)
            obs[f"{name}_n{n}"] = lambda sim=sim, out=out: sim.policy_observe(7, out=out)
    obs_us = {k: [] for k in obs}
    for _ in range(a.rounds):
        for k, f in obs.items():
            obs_us[k].append(events_ms(f, 2000) * 1e3)
    res["policy_observe_us"] = {k: {"runs": v, "median": statistics.median(v)} for k, v in obs_us.items()}

    # (b) the step in a graph of T, with and without the table's row
    arms = {"step": step_graph(make_sim(N), T, False), "step_policy_observe_dp11": step_graph(make_sim(N, NO_POS), T, True),
            "policy_observe_dp11": step_graph(make_sim(N, NO_POS), T, True, step=False),
            "policy_observe_dp32": step_graph(make_sim(N, WIDE), T, True, step=False)}
    step_us = {k: [] for k in arms}
    for _ in range(a.rounds):
        for k, f in arms.items():
            step_us[k].append(events_ms(f, 20) * 1e3 / T)
    res["graph_step_us"] = {k: {"runs": v, "median": statistics.median(v)} for k, v in step_us.items()}
    del arms

    # (d) whole iterations
    from wheeledlab_b200.learner import PPOConfig, PPOIteration
    from wheeledlab_b200.policy import pack_actor_critic
    its = {}
    for name, table in (("fused_builtin_row", None), ("table_dp11", NO_POS)):
        sim = make_sim(N, table)
        D = sim.policy_width
        mk = lambda out: torch.nn.Sequential(torch.nn.Linear(D, 64), torch.nn.ELU(), torch.nn.Linear(64, 64), torch.nn.ELU(),
                                             torch.nn.Linear(64, out))
        torch.manual_seed(0)
        blob = pack_actor_critic(mk(2), mk(1), torch.ones(2), D, DEV)
        its[name] = PPOIteration(sim, blob, PPOConfig(), T, episode_stats=True).start(0, capture=True)
    it_ms = {k: [] for k in its}
    for _ in range(a.rounds):
        for k, it in its.items():
            it_ms[k].append(events_ms(it.run, 10))
    res["iteration_ms"] = {k: {"runs": v, "median": statistics.median(v)} for k, v in it_ms.items()}
    line = json.dumps(res)
    print(line)
    if a.out:
        Path(a.out).parent.mkdir(parents=True, exist_ok=True)
        with open(a.out, "a") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
