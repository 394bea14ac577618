"""A whole PPO training loop on one GPU (Drift, or Elevation with ``--task elevation``): FusedPolicyRollout -> bootstrap value -> compute_returns -> FusedPPO.update,
one CUDA graph per iteration (learner.PPOIteration), with rsl_rl's default Drift settings (learner.PPOConfig) and the
task's network: [64, 64] ELU for Drift, ReLU for Elevation (its agent cfg, activation="relu").

Prints, per iteration, the mean return of the episodes that ended during it, the learning rate and the losses; the
statistics are read back once per iteration, after the graph replay.

    python tools/ppo_train.py [--task elevation] --envs 4096 --iters 50 [--eager] [--out results.txt]
"""
from __future__ import annotations

import argparse
import sys
import time
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--task", choices=["drift", "elevation"], default="drift")
    ap.add_argument("--envs", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=128, help="rollout length T (num_steps_per_env)")
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--eager", action="store_true", help="run the update outside the graph (the rollout stays one graph)")
    ap.add_argument("--out", default=None, help="also write the log here")
    a = ap.parse_args()
    import wheeledlab_b200 as wl
    from wheeledlab_b200.learner import PPOConfig, PPOIteration
    from wheeledlab_b200.policy import pack_actor_critic
    dev = "cuda:0"
    torch.manual_seed(a.seed)
    make, activation, name = (wl.drift_task, "elu", "Drift") if a.task == "drift" else (wl.elevation_task, "relu", "Elevation")
    sim = wl.WheeledSim(make(num_envs=a.envs, seed=a.seed), dev)
    sim.startup(); sim.reset(None, 0)
    D = sim.obs_dim
    act = torch.nn.ELU if activation == "elu" else torch.nn.ReLU
    mk = lambda out: torch.nn.Sequential(torch.nn.Linear(D, 64), act(), torch.nn.Linear(64, 64), act(), torch.nn.Linear(64, out))
    blob = pack_actor_critic(mk(2), mk(1), torch.ones(2), D, dev)           # init_noise_std = 1.0 (rsl_rl_ppo_cfg.py:13)
    it = PPOIteration(sim, blob, PPOConfig(), a.steps, activation=activation).start(0, capture=not a.eager)
    cur = torch.zeros(a.envs, device=dev)
    lines = [f"# {name} PPO (obs_dim {D}, {activation}), {a.envs} envs x {a.steps} steps, PPOConfig() defaults, seed {a.seed}, "
             f"{'eager update' if a.eager else 'one graph per iteration'}, {torch.cuda.get_device_name(0)}",
             "iter  mean_episode_reward  episodes  learning_rate  value_loss  surrogate  entropy  ms"]
    print(lines[0]); print(lines[1])
    for k in range(a.iters):
        t0 = time.perf_counter()
        stats = it.run()
        slab = it.roll.slab
        ep_sum = torch.zeros((), device=dev); ep_n = torch.zeros((), device=dev)
        done = (slab.terminated | slab.truncated).bool()
        for t in range(a.steps):                                             # returns of the episodes that ended
            cur += slab.rewards[t]
            ep_sum += (cur * done[t]).sum(); ep_n += done[t].sum()
            cur *= ~done[t]
        vals = torch.stack([ep_sum / ep_n.clamp(min=1), ep_n, stats["learning_rate"], stats["value_function"], stats["surrogate"],
                            stats["entropy"]]).tolist()
        ms = (time.perf_counter() - t0) * 1e3
        line = f"{k:4d}  {vals[0]:19.4f}  {int(vals[1]):8d}  {vals[2]:13.3e}  {vals[3]:10.4f}  {vals[4]:9.4f}  {vals[5]:7.4f}  {ms:6.2f}"
        print(line, flush=True)
        lines.append(line)
    if a.out:
        Path(a.out).parent.mkdir(parents=True, exist_ok=True)
        Path(a.out).write_text("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
