"""What the asymmetric actor-critic (DESIGN 6m) costs against the symmetric one, Drift N x T, arms alternating within one run:

(a) one rollout step: ``wl_act_step`` (policy fused into the step) against ``wl_policy_act_asym`` + ``wl_step`` +
    ``wl_critic_observe``, each as a CUDA graph of T steps, CUDA events over the replays;
(b) one PPO update: ``wl_ppo_update`` against ``wl_ppo_update_asym`` at Dc = 14 and 29, CUDA events over eager calls;
(c) one whole iteration graph (rollout, episode statistics, bootstrap, GAE, update): symmetric against asymmetric (Dc = 23:
    the 14 noise-free floats plus friction, mass and damping).

    python tools/asym_bench.py [--envs 4096] [--steps 128] [--rounds 3] --out results.json

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
POLICY = ["root_pos_w", "root_euler_xyz", "base_lin_vel", "base_ang_vel", ("last_action", 1.0)]
TABLES = {14: POLICY, 23: POLICY + ["wheel_friction", "base_mass", "motor_damping"],
          29: POLICY + ["joint_vel", "joint_pos", "wheel_friction", "base_mass", "motor_damping"]}


def events_ms(fn, reps: int) -> float:
    fn(); torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def nets(dc, D=14):
    mk = lambda nin, out: torch.nn.Sequential(torch.nn.Linear(nin, 64), torch.nn.ELU(), torch.nn.Linear(64, 64), torch.nn.ELU(),
                                              torch.nn.Linear(64, out))
    return mk(D, 2), mk(dc or D, 1), torch.ones(2)


def make_iteration(n, T, dc):
    import wheeledlab_b200 as wl
    from wheeledlab_b200.learner import PPOConfig, PPOIteration
    from wheeledlab_b200.policy import pack_actor_critic
    sim = wl.WheeledSim(wl.drift_task(num_envs=n, seed=3), DEV); sim.startup(); sim.reset(None, 0)
    if dc:
        sim.set_critic_terms(TABLES[dc])
    torch.manual_seed(0)
    blob = pack_actor_critic(*nets(dc), 14, DEV, critic_obs_dim=dc)
    return PPOIteration(sim, blob, PPOConfig(), T, episode_stats=True, critic=bool(dc)).start(0, capture=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=128)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("asym_bench needs a CUDA device: nothing is measured without one")
    import wheeledlab_b200 as wl
    from wheeledlab_b200.learner import FusedPPO, PPOConfig, compute_returns
    from wheeledlab_b200.policy import FusedPolicyRollout, critic_value, pack_actor_critic
    N, T = a.envs, a.steps
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    res = {"gpu": smi, "envs": N, "steps": T, "rounds": a.rounds}

    # (a) rollout step, graphs of T
    rolls = {}
    for name, dc in (("act_step", None), ("asym_dc23", 23), ("asym_dc29", 29)):
        sim = wl.WheeledSim(wl.drift_task(num_envs=N, seed=3), DEV); sim.startup(); sim.reset(None, 0)
        if dc:
            sim.set_critic_terms(TABLES[dc])
        blob = pack_actor_critic(*nets(dc), 14, DEV, critic_obs_dim=dc)
        rolls[name] = FusedPolicyRollout(sim, blob, T, critic=bool(dc)).capture(0)
    step_us = {k: [] for k in rolls}
    for _ in range(a.rounds):
        for k, r in rolls.items():
            step_us[k].append(events_ms(r.run, 20) * 1e3 / T)
    res["rollout_step_us"] = {k: {"runs": v, "median": statistics.median(v)} for k, v in step_us.items()}

    # (b) the update on a real slab
    ups = {}
    for name, dc in (("sym", None), ("asym_dc14", 14), ("asym_dc29", 29)):
        r = rolls["act_step"] if dc is None else None
        if dc is not None:
            sim = wl.WheeledSim(wl.drift_task(num_envs=N, seed=3), DEV); sim.startup(); sim.reset(None, 0)
            sim.set_critic_terms(TABLES[dc])
            r = FusedPolicyRollout(sim, pack_actor_critic(*nets(dc), 14, DEV, critic_obs_dim=dc), T, critic=True).capture(0)
        slab = r.run()
        last = critic_value(r.blob, 14, r.cobs0 if dc else r.obs0, critic_obs_dim=dc)
        ret, adv = compute_returns(slab.rewards, slab.values, last, slab.terminated | slab.truncated, 0.99, 0.95, time_outs=slab.truncated)
        perm = torch.randperm(T * N, device=DEV)
        ppo = FusedPPO(r.blob.clone(), 14, PPOConfig(), critic_obs_dim=dc)
        ups[name] = lambda ppo=ppo, slab=slab, ret=ret, adv=adv, perm=perm: ppo.update(slab, ret, adv, perm)
    up_ms = {k: [] for k in ups}
    for _ in range(a.rounds):
        for k, f in ups.items():
            up_ms[k].append(events_ms(f, 5))
    res["ppo_update_ms"] = {k: {"runs": v, "median": statistics.median(v)} for k, v in up_ms.items()}
    del rolls, ups

    # (c) whole iterations
    its = {"sym": make_iteration(N, T, None), "asym_dc23": make_iteration(N, T, 23)}
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
