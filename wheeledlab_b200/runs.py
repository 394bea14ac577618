"""A training run's directory, as ``tools/ppo_train.py --log-dir`` writes it and ``tools/play_policy.py -p`` reads it:
``run.json`` (the task, num_envs, seed and rsl_rl agent cfg: the counterpart of the reference's ``run_config.pkl``),
``models/model_{it}.pt`` (rsl_rl checkpoints) and ``playback/`` (play_policy.py's rollouts)."""
from __future__ import annotations

import json
import os
import re

from .tasks import GYM_IDS

RUN_CONFIG = "run.json"
_MODEL = re.compile(r"model_(\d+)\.pt$")


def agent_cfg(activation: str, steps: int = 128, save_interval: int = 50) -> dict:
    """The reference's agent cfg (``MushrPPORunnerCfg().to_dict()`` of the task's rsl_rl_ppo_cfg.py), the fields the runner reads."""
    from dataclasses import asdict
    from .learner import PPOConfig
    return {"num_steps_per_env": steps, "save_interval": save_interval, "empirical_normalization": False,
            "policy": {"class_name": "ActorCritic", "init_noise_std": 1.0, "actor_hidden_dims": [64, 64],
                       "critic_hidden_dims": [64, 64], "activation": activation},
            "algorithm": {"class_name": "PPO", **asdict(PPOConfig())}}


def distillation_agent_cfg(activation: str, steps: int = 128, save_interval: int = 50) -> dict:
    """rsl_rl's StudentTeacher + Distillation agent cfg [UPSTREAM-RECALL] with rsl-rl-lib 2.3's defaults and the task's
    activation: the agent cfg of a run that distils a teacher (``tools/ppo_train.py --teacher``)."""
    from dataclasses import asdict
    from .learner import DistillationConfig
    return {"num_steps_per_env": steps, "save_interval": save_interval, "empirical_normalization": False,
            "policy": {"class_name": "StudentTeacher", "init_noise_std": 0.1, "noise_std_type": "scalar",
                       "student_hidden_dims": [64, 64], "teacher_hidden_dims": [64, 64], "activation": activation},
            "algorithm": {"class_name": "Distillation", **asdict(DistillationConfig())}}


def task_activation(task: str) -> str:
    """The hidden activation of the reference's agent cfg for `task` (a gym id or task name): ReLU for Elevation and Visual,
    ELU for the Drift family."""
    name = GYM_IDS.get(task, task)
    return "relu" if name in ("elevation", "visual", "visual_random") else "elu"


def save_run_config(log_dir: str, task: str, num_envs: int, seed: int, agent: dict, policy_terms=None, row_terms=None,
                    teacher_terms=None) -> str:
    """`policy_terms`: the env's policy observation table (``(name, library term, noise, clip, scale)`` as
    ``TaskSpec.policy_terms`` holds it), so that playback observes what the policy was trained on; None: the built-in row.
    `row_terms`: the Elevation / Visual env's row terms in the same form (``env.row_terms``, ``TaskSpec.row_terms``): their
    clips and scales change the policy's input even where playback draws no noise.  `teacher_terms`: a distillation run's
    teacher group (``env.set_teacher_observation``'s ``(name, term, params)`` list), which its runner needs to load."""
    os.makedirs(log_dir, exist_ok=True)
    path = os.path.join(log_dir, RUN_CONFIG)
    cfg = {"task": task, "num_envs": int(num_envs), "seed": int(seed), "agent_cfg": agent}
    if policy_terms:
        cfg["policy_terms"] = [list(t) for t in policy_terms]
    if row_terms:
        cfg["row_terms"] = [list(t) for t in row_terms]
    if teacher_terms:
        cfg["teacher_terms"] = [[name, fn, dict(params)] for name, fn, params in teacher_terms]
    with open(path, "w") as f:
        json.dump(cfg, f, indent=1)
    return path


def load_run_config(run_path: str) -> dict | None:
    """The run's ``run.json`` as a dict, or None when the run has none."""
    path = os.path.join(run_path, RUN_CONFIG)
    if not os.path.exists(path):
        return None
    with open(path) as f:
        cfg = json.load(f)
    if not isinstance(cfg, dict) or not {"task", "agent_cfg"} <= set(cfg):
        raise ValueError(f"{path}: not a run config (task, num_envs, seed, agent_cfg)")
    return cfg


def checkpoint_path(run_path: str, checkpoint: int | None = None) -> str:
    """``models/model_{checkpoint}.pt`` of the run, or the one with the highest iteration when `checkpoint` is None."""
    models = os.path.join(run_path, "models")
    if checkpoint is not None:
        path = os.path.join(models, f"model_{int(checkpoint)}.pt")
        if not os.path.isfile(path):
            raise FileNotFoundError(f"checkpoint {checkpoint}: {path} does not exist")
        return path
    its = sorted(int(m.group(1)) for f in (os.listdir(models) if os.path.isdir(models) else []) if (m := _MODEL.fullmatch(f)))
    if not its:
        raise FileNotFoundError(f"no checkpoint model_<iteration>.pt in {models}")
    return os.path.join(models, f"model_{its[-1]}.pt")
