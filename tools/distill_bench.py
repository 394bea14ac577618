"""What a distillation iteration (DESIGN 6t) costs against a PPO iteration of the same task and size, arms alternating
within one run: each is its one CUDA graph (rollout, episode statistics, update) replayed, timed with CUDA events.

    Drift      4096 envs x T: PPOIteration (wl_act_step, GAE, wl_ppo_update) against DistillationIteration (wl_actor_mean of
               a 15-float teacher row, wl_policy_act_elu, wl_step, wl_critic_observe, wl_distill_update; ELU)
    Elevation  1024 and 4096 envs x T: PPOIteration (ReLU) against DistillationIteration with a 698-float row-critic teacher

The student and teacher are freshly initialised; only time is measured.  Distillation uses rsl_rl's defaults (1 epoch,
gradient_length 15, no clip); PPO uses PPOConfig().

    python tools/distill_bench.py [--steps 128] [--rounds 3] [--reps 5] --out results.json

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
DRIFT_TEACHER = ["root_euler_xyz", "base_lin_vel", "base_ang_vel", ("last_action", 1.0), "wheel_friction"]      # 15 floats
ELEV_TEACHER = [("goal_relative_xyz", None, (-5.0, 5.0), None), ("root_euler_xyz", None, None, None),
                ("base_lin_vel", None, (-10.0, 10.0), None), ("base_ang_vel", None, (-10.0, 10.0), None),
                ("last_action", None, (-1.0, 1.0), None), ("world_height_map", None, (-10.0, 10.0), None)]
ELEV_EXTRA = ["wheel_friction", "base_mass", "motor_damping"]


def events_ms(fn, reps: int) -> float:
    fn(); torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def _mlp(nin, out, act):
    a = torch.nn.ELU if act == "elu" else torch.nn.ReLU
    return torch.nn.Sequential(torch.nn.Linear(nin, 64), a(), torch.nn.Linear(64, 64), a(), torch.nn.Linear(64, out))


def _sim(task, n):
    import wheeledlab_b200 as wl
    spec = wl.drift_task(num_envs=n, seed=3) if task == "drift" else wl.elevation_task(num_envs=n, seed=3)
    sim = wl.WheeledSim(spec, DEV)
    sim.startup(); sim.reset(None, 0)
    return sim


def arms(task, n, T):
    from wheeledlab_b200.learner import DistillationIteration, PPOConfig, PPOIteration
    from wheeledlab_b200.policy import pack_actor_critic
    act = "elu" if task == "drift" else "relu"
    torch.manual_seed(0)
    sim = _sim(task, n)
    D = sim.obs_dim
    ppo = PPOIteration(sim, pack_actor_critic(_mlp(D, 2, act), _mlp(D, 1, act), torch.ones(2), D, DEV), PPOConfig(), T, act,
                       episode_stats=True).start(0, capture=True)
    sim2 = _sim(task, n)
    Dt = sim2.set_critic_terms(DRIFT_TEACHER) if task == "drift" else sim2.set_row_critic(ELEV_TEACHER, ELEV_EXTRA)
    student = pack_actor_critic(_mlp(D, 2, act), _mlp(D, 1, act), torch.ones(2), D, DEV)
    teacher = pack_actor_critic(_mlp(Dt, 2, act), _mlp(Dt, 1, act), torch.ones(2), Dt, DEV)
    dist = DistillationIteration(sim2, student, teacher, None, T, act).start(0, capture=True)
    return ppo, dist, Dt


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=128)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", required=True)
    a = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("distill_bench.py: no CUDA device")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip()
    out = {"gpu": q, "T": a.steps, "rounds": a.rounds, "reps": a.reps, "cases": []}
    for task, n in (("drift", 4096), ("elevation", 1024), ("elevation", 4096)):
        ppo, dist, Dt = arms(task, n, a.steps)
        ppo_ms, dist_ms = [], []
        for _ in range(a.rounds):
            ppo_ms.append(events_ms(ppo.run, a.reps))
            dist_ms.append(events_ms(dist.run, a.reps))
        case = {"task": task, "envs": n, "teacher_width": Dt, "ppo_iteration_ms": ppo_ms, "distill_iteration_ms": dist_ms,
                "ppo_median_ms": statistics.median(ppo_ms), "distill_median_ms": statistics.median(dist_ms),
                "distill_losses_finite": bool(torch.isfinite(dist.alg.losses).all())}
        out["cases"].append(case)
        print(json.dumps(case), flush=True)
        del ppo, dist
        torch.cuda.empty_cache()
    Path(a.out).parent.mkdir(parents=True, exist_ok=True)
    Path(a.out).write_text(json.dumps(out, indent=1))
    print(json.dumps({"gpu": q}))


if __name__ == "__main__":
    main()
