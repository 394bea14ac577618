"""What the Elevation asymmetric actor-critic (DESIGN 6s) costs against the symmetric one, arms alternating within one run,
at 1024 envs (the reference RSS_ELEV_CONFIG size) and 4096 envs, T steps per iteration, Gaussian noise on every row column:

(a) the rollout, per step, in its CUDA graph of T steps: symmetric (wl_policy_act, wl_step) against asymmetric
    (wl_policy_act_wide_asym, wl_step, wl_critic_observe);
(b) the second ray cast alone: T device-counter wl_critic_observe calls in one graph, per call;
(c) the PPO update with PPOConfig() on the slab the rollout left: wl_ppo_update_wide against wl_ppo_update_wide_asym;
(d) the whole iteration (rollout, GAE, update) as PPOIteration replays its one graph.
CUDA events throughout.  No learning comparison is made.

    python tools/elev_asym_bench.py [--envs 1024 4096] [--steps 128] [--rounds 3] --out results.json

The card's name, power limit and SM clock are read in the same run and written beside the figures.
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
POLICY = [("goal_relative_xyz", ("gaussian", 0.0, 0.05), None, None), ("root_euler_xyz", ("gaussian", 0.0, 0.05), None, None),
          ("base_lin_vel", ("gaussian", 0.0, 0.1), (-10.0, 10.0), None), ("base_ang_vel", ("gaussian", 0.0, 0.1), (-10.0, 10.0), None),
          ("last_action", ("gaussian", 0.0, 0.05), (-1.0, 1.0), None), ("world_height_map", ("gaussian", 0.0, 0.02), (-10.0, 10.0), None)]
CRITIC = [(fn, None, cl, sc) for fn, _, cl, sc in POLICY]
EXTRA = ["wheel_friction", "base_mass", "motor_damping"]


def events_ms(fn, reps: int) -> float:
    fn(); torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def iteration(n, T, critic):
    import wheeledlab_b200 as wl
    from wheeledlab_b200.learner import PPOConfig, PPOIteration
    from wheeledlab_b200.policy import pack_actor_critic
    spec = wl.elevation_task(num_envs=n, seed=3)
    spec.cfg.enable_corruption = 1
    sim = wl.WheeledSim(spec, DEV)
    sim.set_row_terms(POLICY)
    dc = sim.set_row_critic(CRITIC, EXTRA) if critic else None
    sim.startup(); sim.reset(None, 0)
    torch.manual_seed(0)
    mk = lambda nin, out: torch.nn.Sequential(torch.nn.Linear(nin, 64), torch.nn.ReLU(), torch.nn.Linear(64, 64), torch.nn.ReLU(),
                                              torch.nn.Linear(64, out))
    blob = pack_actor_critic(mk(689, 2), mk(dc or 689, 1), torch.ones(2), 689, DEV, critic_obs_dim=dc)
    it = PPOIteration(sim, blob, PPOConfig(), T, "relu", critic=critic).start(0, capture=True)
    return it


def rollout_graph(it):
    """The iteration's rollout alone, captured as its own graph (the iteration's graph holds it with the update)."""
    from wheeledlab_b200.policy import FusedPolicyRollout
    r = FusedPolicyRollout(it.sim, it.blob, it.T, slab=it.roll.slab, activation="relu", critic=it.critic_obs_dim is not None)
    r.capture(it.T)
    return lambda keep=r: keep.graph.replay()                   # (the rollout owns the buffers its graph writes)


def critic_graph(it):
    sim, T = it.sim, it.T
    out = torch.empty((sim.num_envs, sim.critic_obs_dim), device=DEV)
    g, s = torch.cuda.CUDAGraph(), torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s), torch.cuda.graph(g, stream=s):
        for _ in range(T):
            sim.critic_observe(out=out)
    torch.cuda.current_stream().wait_stream(s)
    return lambda keep=out: g.replay()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, nargs="+", default=[1024, 4096])
    ap.add_argument("--steps", type=int, default=128)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("elev_asym_bench needs a CUDA device: nothing is measured without one")
    T = a.steps
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    res = {"gpu (name, power limit, SM clock, max SM clock)": smi, "steps": T, "rounds": a.rounds, "row_noise": "gaussian, every column",
           "learning_comparison": "not run"}
    for n in a.envs:
        its = {"sym": iteration(n, T, False), "asym": iteration(n, T, True)}
        roll = {k: rollout_graph(v) for k, v in its.items()}
        perm = torch.randperm(n * T, device=DEV)
        for v in its.values():
            v.run(perm)                                         # a slab from this policy for the update arm
        rets = {k: v._returns() for k, v in its.items()}
        upd = {k: (lambda it=v, r=rets[k]: it.ppo.update(it.roll.slab, *r, perm)) for k, v in its.items()}
        whole = {k: (lambda it=v: it.run(perm)) for k, v in its.items()}
        cast = critic_graph(its["asym"])
        runs = {f"{what}_{k}": [] for what in ("rollout_step_us", "update_ms", "iteration_ms") for k in its}
        runs["critic_ray_cast_us"] = []
        for _ in range(a.rounds):
            for k in its:
                runs[f"rollout_step_us_{k}"].append(events_ms(roll[k], 5) * 1e3 / T)
                runs[f"update_ms_{k}"].append(events_ms(upd[k], 3))
                runs[f"iteration_ms_{k}"].append(events_ms(whole[k], 3))
            runs["critic_ray_cast_us"].append(events_ms(cast, 5) * 1e3 / T)
        res[f"envs_{n}"] = {k: {"runs": v, "median": statistics.median(v)} for k, v in runs.items()}
        del its, roll, upd, whole, cast, rets
        torch.cuda.empty_cache()
    line = json.dumps(res)
    print(line)
    if a.out:
        Path(a.out).parent.mkdir(parents=True, exist_ok=True)
        with open(a.out, "a") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
