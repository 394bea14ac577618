"""Play a trained policy and record the data: the reference's ``play_policy.py`` on the fused runner.

    python tools/play_policy.py -p <run-dir> [--checkpoint N] [--steps 200] [-sd] [--play-name NAME]
    python tools/play_policy.py --task Isaac-MushrDriftRL-v0 --policy-path model_50.pt [--log-dir playback/] [-sd]

The checkpoint (``models/model_N.pt`` of the run, the highest iteration unless ``--checkpoint N``) is loaded with
``FusedOnPolicyRunner.load`` (weights only) and played for ``--steps`` steps as ONE CUDA graph of the deterministic
policy: the action is the actor mean (rsl_rl's ``get_inference_policy``), T x ``wl_act_infer_step`` for the Drift family's
ELU network, T x (``wl_actor_mean`` -> ``wl_step``) for the ReLU network of Elevation and Visual.  The task, num_envs, seed
and agent cfg come from the run's ``run.json`` (``tools/ppo_train.py --log-dir``); without one, ``--task`` is needed and
the activation follows the task.  ``-sd`` saves ``{'observations', 'actions'}`` as ``<playback-dir>/<play-name>-rollouts.pt``,
the reference's file.  Prints the mean return and length of the episodes that finished during the playback.  A run trained on
a policy observation table (``policy_terms`` in ``run.json``, DESIGN 6q) plays on an env with the same table, through
``wl_actor_mean`` on the table's row.
"""
from __future__ import annotations

import argparse
import os
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))


def parser() -> argparse.ArgumentParser:
    ap = argparse.ArgumentParser(description="Play a policy in WheeledLab.")
    ap.add_argument("-p", "--run-path", type=str, default=None, help="Path to run folder")
    ap.add_argument("--checkpoint", type=int, default=None, help="Checkpoint to load (models/model_N.pt; default: the highest N)")
    ap.add_argument("--task", type=str, default=None, help="Task name. Overrides run config env if provided")
    ap.add_argument("--policy-path", type=str, default=None, help="Path to policy file.")
    ap.add_argument("--steps", type=int, default=200, help="Length of the playback in steps")
    ap.add_argument("-sd", "--save-data", action="store_true", help="Save episode data")
    ap.add_argument("--video", action="store_true", help="Not supported: there is no viewport to record")
    ap.add_argument("--log-dir", type=str, default="playback/", help="Directory to save logs. If run path is provided, this is ignored.")
    ap.add_argument("--play-name", type=str, default="play-name", help="Name of the playback")
    ap.add_argument("--num-envs", type=int, default=None, help="Number of envs (default: the run's, else the task's)")
    ap.add_argument("--seed", type=int, default=None, help="Env seed (default: the run's, else the task's)")
    return ap


def resolve(args) -> dict:
    """What to play, from the arguments alone (no device): task, checkpoint, playback dir, activation, agent cfg, num_envs,
    seed.  Raises ValueError / FileNotFoundError with the reason."""
    from wheeledlab_b200.runs import agent_cfg, checkpoint_path, load_run_config, task_activation
    if args.video:
        raise ValueError("--video is not supported: env.render() returns None (there is no RTX viewport to record); play without --video")
    if args.steps < 1:
        raise ValueError("--steps must be >= 1")
    if args.run_path is None:
        if args.task is None or args.policy_path is None:
            raise ValueError("Either path to run directory or task/policy must be provided.")
        run_cfg, policy_path, playback_dir = None, args.policy_path, args.log_dir
        if not os.path.isfile(policy_path):
            raise FileNotFoundError(f"--policy-path {policy_path} does not exist")
    else:
        run_cfg = load_run_config(args.run_path)
        policy_path = checkpoint_path(args.run_path, args.checkpoint)
        playback_dir = os.path.join(args.run_path, "playback")
    task = args.task if args.task is not None else (run_cfg or {}).get("task")
    if task is None:
        raise ValueError(f"{args.run_path} has no run.json: pass --task")
    agent = run_cfg["agent_cfg"] if run_cfg is not None else agent_cfg(task_activation(task))
    num_envs = args.num_envs if args.num_envs is not None else (run_cfg or {}).get("num_envs")
    seed = args.seed if args.seed is not None else (run_cfg or {}).get("seed")
    return {"task": task, "policy_path": policy_path, "playback_dir": playback_dir, "agent_cfg": agent, "num_envs": num_envs, "seed": seed,
            "policy_terms": (run_cfg or {}).get("policy_terms")}


def play(r: dict, steps: int, device: str = "cuda:0"):
    """Load the checkpoint and play `steps` steps as one deterministic graph.  Returns (runner, rollout, EpisodeStatistics)."""
    import torch
    import wheeledlab_b200 as wl
    from wheeledlab_b200.learner import EpisodeStatistics, FusedOnPolicyRunner
    from wheeledlab_b200.policy import FusedPolicyRollout
    kw = {k: r[k] for k in ("num_envs", "seed") if r[k] is not None}
    env = wl.make(r["task"], device=device, **kw)
    if r.get("policy_terms"):
        env.set_policy_observation([(name, fn, {"noise": tuple(nz) if nz else None, "clip": cl, "scale": sc})
                                    for name, fn, nz, cl, sc in r["policy_terms"]])
    runner = FusedOnPolicyRunner(env, r["agent_cfg"], device=device)
    runner.load(r["policy_path"], load_optimizer=False)
    env.reset()
    roll = FusedPolicyRollout(env.sim, runner.blob, steps, activation=runner.activation, deterministic=True)
    roll.capture(env.common_step_counter)
    slab = roll.run()
    env.common_step_counter += steps
    env.sim.flush_log()
    stats = EpisodeStatistics(env.num_envs, steps, env.sim.device)
    stats.update(slab.rewards, slab.terminated, slab.truncated)
    torch.cuda.synchronize(env.sim.device)
    return runner, roll, stats


def main(argv=None):
    args = parser().parse_args(argv)
    try:
        r = resolve(args)
    except (ValueError, FileNotFoundError) as e:
        print(f"play_policy.py: error: {e}", file=sys.stderr)
        return 2
    os.makedirs(r["playback_dir"], exist_ok=True)
    print(f"[INFO] Created playback directory: {r['playback_dir']}")
    runner, roll, stats = play(r, args.steps)
    env = runner.env
    print(f"[INFO] Played {r['policy_path']} on {r['task']} ({env.num_envs} envs, {runner.activation}) for {args.steps} steps, "
          f"the actor mean as one CUDA graph")
    if args.save_data:
        from wheeledlab_b200.recording import save_slab
        path = save_slab(r["playback_dir"], args.play_name, roll.slab)
        print(f"[INFO] Saved episode data to: {path}")
    fill, _, fin = stats.counts.tolist()
    mean_return, mean_length = stats.means.tolist()
    if fin:
        print(f"Episodes finished: {fin}; mean return {mean_return:.4f}, mean length {mean_length:.2f} (the last {fill})")
    else:
        print(f"Episodes finished: 0 (no episode ended within {args.steps} steps)")
    print("Done playing policy. Closing environment.")
    env.close()
    return 0


if __name__ == "__main__":
    sys.exit(main())
