"""A whole PPO training job on one GPU through learner.FusedOnPolicyRunner: Drift, Elevation (``--task elevation``) or the
camera Visual task (``--task visual``), with the task's rsl_rl agent cfg (T = 128, [64, 64] ELU for Drift, ReLU for
Elevation and Visual, rsl_rl's PPO settings, save_interval 50).  One CUDA graph per iteration; one read-back per iteration.

Prints, per iteration, the reference runner's Train/mean_reward and Train/mean_episode_length (the last 100 finished
episodes, once there is one), the episodes finished in the iteration, the learning rate, the losses and the iteration time.
``--log-dir`` saves ``models/model_{it}.pt`` every ``--save-interval`` iterations and the run's ``run.json`` (task, num_envs,
seed, agent cfg; what ``tools/play_policy.py -p LOG_DIR`` reads); ``--resume PATH`` continues from one.

    python tools/ppo_train.py [--task elevation|visual] --envs 4096 --iters 50 [--log-dir DIR] [--resume DIR/models/model_25.pt] [--out log.txt]

Under ``torchrun --nproc-per-node=R`` it trains data-parallel (rsl_rl's multi-GPU PPO, DESIGN 6j): ``--envs`` per rank, rank r
simulating envs r * envs .. (r + 1) * envs - 1 of one big run on cuda:LOCAL_RANK; only rank 0 prints and writes.

``--teacher CKPT`` distils instead (rsl_rl's StudentTeacher + Distillation, DESIGN 6t; Drift or Elevation, one GPU): the
env gets a ``teacher`` group of ``--teacher-terms`` (default: the task's policy row terms without noise, so a PPO checkpoint
of the task is a teacher), the PPO checkpoint's actor becomes the teacher, and the student learns on the noisy row.

    python tools/ppo_train.py --task drift --teacher RUN/models/model_500.pt [--teacher-terms root_euler_xyz,...,wheel_friction]
"""
from __future__ import annotations

import argparse
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))

TASKS = {"drift": ("Isaac-MushrDriftRL-v0", "elu", "Drift"), "elevation": ("Isaac-MushrElevationRL-v0", "relu", "Elevation"),
         "visual": ("Isaac-MushrVisualRL-v0", "relu", "Visual (camera)")}
# each task's policy row terms in row order: the default teacher row, noise-free (the map of Elevation clipped, as it must be)
TEACHER_TERMS = {"drift": "root_pos_w,root_euler_xyz,base_lin_vel,base_ang_vel,last_action",
                 "elevation": "goal_relative_xyz,root_euler_xyz,base_lin_vel,base_ang_vel,last_action,world_height_map"}


def teacher_group(task: str, names: str | None) -> list:
    """`--teacher-terms` as env.set_teacher_observation's list; the Elevation height map gets the clip a row critic needs."""
    if task not in TEACHER_TERMS:
        raise SystemExit(f"ppo_train.py: --teacher: distillation covers the Drift family and Elevation, not {task}")
    out = []
    for name in (names or TEACHER_TERMS[task]).split(","):
        params = {"clip": (-10.0, 10.0)} if name == "world_height_map" else {"clip": (-1.0, 1.0)} if name == "last_action" else {}
        out.append((name, name, params))
    return out


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
    ap.add_argument("--reset-events", default="", help="DR events redrawn at every reset (mode='reset'), comma-separated: "
                                                        "material, actuator_gains, base_mass, wheel_mass")
    ap.add_argument("--teacher", default=None, help="distil the actor of this PPO checkpoint into a student (StudentTeacher + Distillation)")
    ap.add_argument("--teacher-terms", default=None, help="the teacher row's terms, comma-separated (default: the policy row's, noise-free)")
    a = ap.parse_args()
    import wheeledlab_b200 as wl
    from wheeledlab_b200.learner import FusedOnPolicyRunner
    from wheeledlab_b200.runs import agent_cfg, distillation_agent_cfg, save_run_config
    import os
    rank, world = int(os.environ.get("RANK", "0")), int(os.environ.get("WORLD_SIZE", "1"))
    dev = f"cuda:{int(os.environ.get('LOCAL_RANK', '0'))}"
    torch.manual_seed(a.seed)
    task_id, activation, name = TASKS[a.task]
    env = wl.make(task_id, device=dev, num_envs=a.envs, seed=a.seed, env_id_offset=rank * a.envs)
    events = [e for e in a.reset_events.split(",") if e]
    if events:
        env.sim.set_reset_events(**{e: True for e in events})
    teacher = teacher_group(a.task, a.teacher_terms) if a.teacher else None
    if teacher:
        env.set_teacher_observation(teacher)
    agent = (distillation_agent_cfg if teacher else agent_cfg)(activation, a.steps, a.save_interval)
    runner = FusedOnPolicyRunner(env, agent, log_dir=a.log_dir, device=dev)
    if a.log_dir and rank == 0:
        save_run_config(a.log_dir, task_id, a.envs, a.seed, agent, teacher_terms=teacher)
    if teacher:
        runner.load(a.teacher)                                # the PPO checkpoint's actor: the teacher (not resumed)
        name += f" distillation of {Path(a.teacher).name} (teacher row {env.sim.critic_obs_dim})"
    head = (f"# {name} {'' if teacher else 'PPO '}(obs_dim {env.sim.obs_dim}, {activation}), {a.envs} envs x {a.steps} steps" + (f" x {world} ranks" if world > 1 else "")
            + f", rsl_rl agent cfg, seed {a.seed}" + (f", reset-mode DR: {', '.join(events)}" if events else "")
            + f", one graph per iteration, {torch.cuda.get_device_name(dev)}")
    if a.resume:
        runner.load(a.resume)
        env.common_step_counter = runner.current_learning_iteration * a.steps     # continue the curriculum where it was
        head += f"; resumed from {Path(a.resume).name} at iteration {runner.current_learning_iteration}"
    losses = "behavior" if teacher else "value_loss  surrogate  entropy"
    lines = [head, f"iter  Train/mean_reward  Train/mean_episode_length  finished  learning_rate  {losses}  ms"]
    if rank == 0:
        print(lines[0]); print(lines[1])

    def log(it, s):
        mr, ml = s.get("Train/mean_reward", float("nan")), s.get("Train/mean_episode_length", float("nan"))
        ms = a.steps * a.envs * world / s["Perf/total_fps"] * 1e3
        loss = (f"{s['Loss/behavior']:8.5f}" if teacher else
                f"{s['Loss/value_function']:10.4f}  {s['Loss/surrogate']:9.4f}  {s['Loss/entropy']:7.4f}")
        line = (f"{it:4d}  {mr:17.4f}  {ml:25.2f}  {s['Episodes/finished']:8d}  {s['Loss/learning_rate']:13.3e}  "
                f"{loss}  {ms:6.2f}")
        print(line, flush=True)
        lines.append(line)

    runner.callback = log
    runner.learn(a.iters)
    if a.out and rank == 0:
        Path(a.out).parent.mkdir(parents=True, exist_ok=True)
        Path(a.out).write_text("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
