"""A whole PPO training job on one GPU through learner.FusedOnPolicyRunner: Drift, Elevation (``--task elevation``) or the
camera Visual task (``--task visual``), with the task's rsl_rl agent cfg (T = 128, [64, 64] ELU for Drift, ReLU for
Elevation and Visual, rsl_rl's PPO settings, save_interval 50).  One CUDA graph per iteration; one read-back per iteration.

Prints, per iteration, the reference runner's Train/mean_reward and Train/mean_episode_length (the last 100 finished
episodes, once there is one), the episodes finished in the iteration, the learning rate, the losses and the iteration time.
``--log-dir`` saves ``models/model_{it}.pt`` every ``--save-interval`` iterations; ``--resume PATH`` continues from one.

    python tools/ppo_train.py [--task elevation|visual] --envs 4096 --iters 50 [--log-dir DIR] [--resume DIR/models/model_25.pt] [--out log.txt]
"""
from __future__ import annotations

import argparse
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))

TASKS = {"drift": ("Isaac-MushrDriftRL-v0", "elu", "Drift"), "elevation": ("Isaac-MushrElevationRL-v0", "relu", "Elevation"),
         "visual": ("Isaac-MushrVisualRL-v0", "relu", "Visual (camera)")}


def agent_cfg(activation: str, steps: int, save_interval: int) -> dict:
    """The reference's agent cfg (``MushrPPORunnerCfg().to_dict()`` of the task's rsl_rl_ppo_cfg.py), the fields the runner reads."""
    from dataclasses import asdict
    from wheeledlab_b200.learner import PPOConfig
    return {"num_steps_per_env": steps, "save_interval": save_interval, "empirical_normalization": False,
            "policy": {"class_name": "ActorCritic", "init_noise_std": 1.0, "actor_hidden_dims": [64, 64],
                       "critic_hidden_dims": [64, 64], "activation": activation},
            "algorithm": {"class_name": "PPO", **asdict(PPOConfig())}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--task", choices=sorted(TASKS), default="drift")
    ap.add_argument("--envs", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=128, help="rollout length T (num_steps_per_env)")
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--save-interval", type=int, default=50)
    ap.add_argument("--log-dir", default=None, help="checkpoints go to LOG_DIR/models/model_{it}.pt")
    ap.add_argument("--resume", default=None, help="checkpoint to continue from (its iteration, weights and Adam state)")
    ap.add_argument("--out", default=None, help="also write the log here")
    a = ap.parse_args()
    import wheeledlab_b200 as wl
    from wheeledlab_b200.learner import FusedOnPolicyRunner
    dev = "cuda:0"
    torch.manual_seed(a.seed)
    task_id, activation, name = TASKS[a.task]
    env = wl.make(task_id, device=dev, num_envs=a.envs, seed=a.seed)
    runner = FusedOnPolicyRunner(env, agent_cfg(activation, a.steps, a.save_interval), log_dir=a.log_dir, device=dev)
    head = (f"# {name} PPO (obs_dim {env.sim.obs_dim}, {activation}), {a.envs} envs x {a.steps} steps, rsl_rl agent cfg, seed {a.seed}, "
            f"one graph per iteration, {torch.cuda.get_device_name(0)}")
    if a.resume:
        runner.load(a.resume)
        env.common_step_counter = runner.current_learning_iteration * a.steps     # continue the curriculum where it was
        head += f"; resumed from {Path(a.resume).name} at iteration {runner.current_learning_iteration}"
    lines = [head, "iter  Train/mean_reward  Train/mean_episode_length  finished  learning_rate  value_loss  surrogate  entropy  ms"]
    print(lines[0]); print(lines[1])

    def log(it, s):
        mr, ml = s.get("Train/mean_reward", float("nan")), s.get("Train/mean_episode_length", float("nan"))
        ms = a.steps * a.envs / s["Perf/total_fps"] * 1e3
        line = (f"{it:4d}  {mr:17.4f}  {ml:25.2f}  {s['Episodes/finished']:8d}  {s['Loss/learning_rate']:13.3e}  "
                f"{s['Loss/value_function']:10.4f}  {s['Loss/surrogate']:9.4f}  {s['Loss/entropy']:7.4f}  {ms:6.2f}")
        print(line, flush=True)
        lines.append(line)

    runner.callback = log
    runner.learn(a.iters)
    if a.out:
        Path(a.out).parent.mkdir(parents=True, exist_ok=True)
        Path(a.out).write_text("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
