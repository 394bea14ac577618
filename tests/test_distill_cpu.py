"""Distillation without a GPU (DESIGN 6t): the runner's settings for rsl_rl's StudentTeacher + Distillation and each of its
refusals by name, the lowering of a ``teacher`` observation group on the Drift family and Elevation, the StudentTeacher
state dict round trip and a PPO checkpoint loading as the teacher alone, and wl_distill_update refusing malformed calls
before any launch (pointers that are never dereferenced, and the Python layers with the library replaced by a stub)."""
import ctypes as C
import sys
from pathlib import Path
from types import SimpleNamespace

import pytest
import torch

ROOT = Path(__file__).resolve().parent.parent
DRIFT = {"num_steps_per_env": 32, "save_interval": 1, "empirical_normalization": False,
         "policy": {"class_name": "StudentTeacher", "init_noise_std": 0.8, "noise_std_type": "scalar", "student_hidden_dims": [64, 64],
                    "teacher_hidden_dims": [64, 64], "activation": "elu"},
         "algorithm": {"class_name": "Distillation", "num_learning_epochs": 2, "gradient_length": 10, "learning_rate": 5e-4,
                       "max_grad_norm": 1.0, "loss_type": "mse"}}


class _NoLaunch:
    """Stands in for the library: any call fails the test (an argument check is missing if one is reached)."""

    def __getattr__(self, name):
        def launch(*args, **kwargs):
            pytest.fail(f"{name} was reached: the call should have been refused before any launch")
        return launch


def _with(**change):
    cfg = {k: dict(v) if isinstance(v, dict) else v for k, v in DRIFT.items()}
    for part, kv in change.items():
        cfg[part].update(kv)
    return cfg


def test_runner_settings_for_student_teacher_distillation():
    from wheeledlab_b200.learner import DistillationConfig, FusedOnPolicyRunner
    s = FusedOnPolicyRunner.settings(DRIFT)
    assert s.distillation and (s.num_steps_per_env, s.save_interval, s.activation, s.init_noise_std) == (32, 1, "elu", 0.8)
    assert s.alg_cfg == DistillationConfig(num_learning_epochs=2, gradient_length=10, learning_rate=5e-4, max_grad_norm=1.0)
    # rsl-rl-lib 2.3's defaults for what the cfg leaves out
    bare = FusedOnPolicyRunner.settings({**DRIFT, "algorithm": {"class_name": "Distillation"}})
    assert bare.alg_cfg == DistillationConfig(1, 15, 1e-3, None, "mse")
    assert FusedOnPolicyRunner.settings(_with(policy={"activation": "relu"})).activation == "relu"


@pytest.mark.parametrize("change,match", [
    (dict(policy={"class_name": "ActorCriticRecurrent"}), "ActorCriticRecurrent"),
    (dict(algorithm={"class_name": "PPO"}), "StudentTeacher \\+ PPO"),
    (dict(policy={"class_name": "StudentTeacherRecurrent"}), "StudentTeacherRecurrent"),
    (dict(algorithm={"loss_type": "huber"}), "loss_type='huber'"),
    (dict(policy={"noise_std_type": "log"}), "noise_std_type='log'"),
    (dict(policy={"student_hidden_dims": [128, 64]}), "\\[128, 64\\]"),
    (dict(policy={"teacher_hidden_dims": [256, 256, 256]}), "\\[256, 256, 256\\]"),
], ids=["recurrent", "student-teacher-ppo", "recurrent-student", "huber", "log-std", "student-dims", "teacher-dims"])
def test_runner_refuses_what_distillation_cannot_run(change, match):
    from wheeledlab_b200.learner import FusedOnPolicyRunner
    with pytest.raises(NotImplementedError, match=match):
        FusedOnPolicyRunner.settings(_with(**change))


def _env(teacher=True, device="cuda:0", **extra):
    sim = SimpleNamespace(device=device, num_envs=64, obs_dim=14, policy_width=14, critic_obs_dim=9 if teacher else 0,
                          cfg=SimpleNamespace(env_id_offset=0))
    return SimpleNamespace(sim=sim, _teacher_terms=[("mu", "wheel_friction", {})] if teacher else [], **extra)


@pytest.mark.parametrize("env,world,match", [
    (dict(teacher=False), 1, "teacher observation group"),
    (dict(_py_rewards=[("r", None, 1.0, {})]), 1, "Python terms or device terms"),
    (dict(_dev_terms=[object()], device_log_names=["Episode_Reward/x"]), 1, "Python terms or device terms"),
    (dict(), 2, "data-parallel"),
], ids=["no-teacher", "python-terms", "device-terms", "data-parallel"])
def test_runner_refuses_distillation_it_cannot_run_before_any_launch(monkeypatch, env, world, match):
    from wheeledlab_b200 import learner
    monkeypatch.setattr(learner, "lib", _NoLaunch())
    monkeypatch.setenv("WORLD_SIZE", str(world))
    exc = ValueError if match == "teacher observation group" else NotImplementedError
    with pytest.raises(exc, match=match):
        learner.FusedOnPolicyRunner(_env(**env), DRIFT, device="cuda:0")


@pytest.fixture(scope="module")
def ref_registry():
    if str(ROOT / "shims") not in sys.path:
        sys.path.insert(0, str(ROOT / "shims"))
    import recorded_cfgs
    return recorded_cfgs.load()


def _group(**terms):
    from isaaclab.managers import ObservationTermCfg
    g = SimpleNamespace(concatenate_terms=True, enable_corruption=False)
    for k, v in terms.items():
        setattr(g, k, v if hasattr(v, "func") else ObservationTermCfg(func=v))
    return g


def test_compat_lowers_a_drift_teacher_group_as_a_critic_table(ref_registry):
    from wheeledlab_b200 import privileged
    from wheeledlab_b200.compat import spec_from_reference_cfg
    cfg = ref_registry["Isaac-MushrDriftRL-v0"]["cfgs"]["env_cfg_entry_point"]()
    cfg.scene.num_envs = 16
    plain = spec_from_reference_cfg(cfg, device_terms=True)
    cfg.observations.teacher = _group(friction=privileged.wheel_friction, mass=privileged.base_mass)
    spec = spec_from_reference_cfg(cfg, device_terms=True)
    assert spec.teacher_terms == [("friction", "wheel_friction", 0.0), ("mass", "base_mass", 0.0)]
    assert spec.critic_terms == [] and spec.row_teacher == [] and bytes(spec.cfg) == bytes(plain.cfg)
    assert spec_from_reference_cfg(cfg).teacher_terms == []             # without device_terms the group is not read
    cfg.observations.critic = _group(friction=privileged.wheel_friction)
    with pytest.raises(NotImplementedError, match="critic observation group or a teacher observation group"):
        spec_from_reference_cfg(cfg, device_terms=True)


def test_compat_lowers_an_elevation_teacher_group_as_a_row_critic(ref_registry):
    from isaaclab.managers import ObservationTermCfg
    from wheeledlab_b200 import privileged
    from wheeledlab_b200.compat import spec_from_reference_cfg
    cfg = ref_registry["Isaac-MushrElevationRL-v0"]["cfgs"]["env_cfg_entry_point"]()
    cfg.scene.num_envs = 16
    g = SimpleNamespace(concatenate_terms=True, enable_corruption=False)
    for name in vars(cfg.observations.policy):
        t = getattr(cfg.observations.policy, name)
        if hasattr(t, "func"):
            setattr(g, name, ObservationTermCfg(func=t.func, params=dict(t.params or {}), clip=getattr(t, "clip", None)))
    g.mu = ObservationTermCfg(func=privileged.wheel_friction)
    cfg.observations.teacher = g
    spec = spec_from_reference_cfg(cfg, device_terms=True)
    assert [fn for _, fn, _ in spec.row_teacher] == ["goal_relative_xyz", "root_euler_xyz", "base_lin_vel", "base_ang_vel",
                                                     "last_action", "world_height_map", "wheel_friction"]
    assert spec.row_critic == [] and spec.teacher_terms == []
    g.mu = ObservationTermCfg(func=lambda env: None)
    with pytest.raises(NotImplementedError, match="term mu"):
        spec_from_reference_cfg(cfg, device_terms=True)


def test_compat_refuses_a_visual_teacher_group_by_name(ref_registry):
    from wheeledlab_b200 import privileged
    from wheeledlab_b200.compat import spec_from_reference_cfg
    cfg = ref_registry["Isaac-MushrVisualRL-v0"]["cfgs"]["env_cfg_entry_point"]()
    cfg.scene.num_envs = 16
    cfg.observations.teacher = _group(friction=privileged.wheel_friction)
    with pytest.raises(NotImplementedError, match="teacher observation group on the Visual task"):
        spec_from_reference_cfg(cfg, device_terms=True)


def _blobs(D=14, Dt=9, seed=0):
    from wheeledlab_b200.policy import blob_layout
    g = torch.Generator().manual_seed(seed)
    s = torch.randn(blob_layout(D)[1], generator=g)
    t = torch.randn(blob_layout(Dt)[1], generator=g)
    return s, t


def test_student_teacher_state_dict_round_trip():
    from wheeledlab_b200.policy import blob_layout, load_student_teacher_state_dict, student_teacher_state_dict
    for D, Dt in ((14, 9), (14, 16), (689, 690)):
        s, t = _blobs(D, Dt)
        sd = student_teacher_state_dict(s, D, t, Dt)
        assert list(sd) == [f"{n}.{k}.{w}" for n in ("student", "teacher") for k in (0, 2, 4) for w in ("weight", "bias")] + ["std"]
        assert sd["student.0.weight"].shape == (64, D) and sd["teacher.0.weight"].shape == (64, Dt) and sd["student.4.weight"].shape == (2, 64)
        s2, t2 = torch.zeros_like(s), torch.zeros_like(t)
        assert load_student_teacher_state_dict(sd, D, Dt, s2, t2) is True
        assert student_teacher_state_dict(s2, D, t2, Dt).keys() == sd.keys()
        for k, v in student_teacher_state_dict(s2, D, t2, Dt).items():
            assert torch.equal(v, sd[k]), k
        o, _ = blob_layout(D)
        assert (s2[o[6]:o[12]] == 0).all()                                # the student's critic blocks are not written


def test_a_ppo_checkpoint_loads_as_the_teacher_only():
    from wheeledlab_b200.policy import actor_critic_state_dict, load_student_teacher_state_dict, student_teacher_state_dict
    s, t = _blobs()
    ppo = actor_critic_state_dict(torch.randn_like(t), 9)                  # a PPO run whose actor read the 9-float teacher row
    s2, t2 = s.clone(), torch.zeros_like(t)
    assert load_student_teacher_state_dict(ppo, 14, 9, s2, t2) is False
    assert torch.equal(s2, s)                                             # the student is left as it was
    got = student_teacher_state_dict(s2, 14, t2, 9)
    for k in (0, 2, 4):
        for w in ("weight", "bias"):
            assert torch.equal(got[f"teacher.{k}.{w}"], ppo[f"actor.{k}.{w}"])
    wrong = actor_critic_state_dict(torch.randn(len(s)), 14)              # an actor over the 14-float policy row
    t3 = t2.clone()
    with pytest.raises(ValueError, match="actor.0.weight is \\(64, 14\\).*teacher row of 9"):
        load_student_teacher_state_dict(wrong, 14, 9, s2, t3)
    assert torch.equal(t3, t2)
    with pytest.raises(ValueError, match="neither"):
        load_student_teacher_state_dict({"std": torch.ones(2)}, 14, 9, s2, t3)


FAKE = 1 << 20                                     # 256-byte aligned, never dereferenced


def _update(obs_dim=14, epochs=1, G=15, mgn=1.0, T=32, N=64, activation=0, null=None, ptrs=None, ws_bytes=1 << 30):
    import wheeledlab_b200 as wl
    from wheeledlab_b200._lib import WlDistillParams
    p = WlDistillParams(obs_dim, epochs, G, mgn)
    args = [C.byref(p), FAKE, FAKE + (1 << 12), T, N, activation, FAKE + (2 << 12), FAKE + (3 << 12), FAKE + (4 << 12),
            FAKE + (5 << 12), FAKE + (6 << 12), ws_bytes, None]
    for i, v in (ptrs or {}).items():
        args[i] = v
    if null is not None:
        args[null] = None
    return wl.lib.wl_distill_update(*args), wl.lib.wl_last_error().decode()


REFUSALS = [
    ("null params", dict(null=0), "null params"),
    ("null obs", dict(null=1), "null d_obs"),
    ("null teacher actions", dict(null=2), "null d_obs / d_teacher_actions"),
    ("null blob", dict(null=6), "null d_obs"),
    ("null state", dict(null=9), "null d_obs"),
    ("null workspace", dict(null=10), "null d_obs"),
    ("unknown activation", dict(activation=2), "activation must be"),
    ("ELU beyond 16", dict(obs_dim=17), "obs_dim <= 16"),
    ("obs_dim 0", dict(obs_dim=0, activation=1), "obs_dim must be in 1..4096"),
    ("obs_dim 4097", dict(obs_dim=4097, activation=1), "obs_dim must be in 1..4096"),
    ("no epochs", dict(epochs=0), "num_learning_epochs must be >= 1"),
    ("gradient length 0", dict(G=0), "gradient_length must be >= 1"),
    ("T < gradient_length", dict(T=14, G=15), "T must be >= gradient_length"),
    ("N 0", dict(N=0), "T and N must be >= 1"),
    ("misaligned blob", dict(ptrs={6: FAKE + 4}), "16-byte aligned"),
    ("misaligned workspace", dict(ptrs={10: FAKE + 16}), "256-byte aligned"),
    ("misaligned teacher actions", dict(ptrs={2: FAKE + 4}), "d_teacher_actions 8-byte"),
]


@pytest.mark.parametrize("kw,match", [c[1:] for c in REFUSALS], ids=[c[0] for c in REFUSALS])
def test_distill_update_refuses_before_any_launch(kw, match):
    rc, msg = _update(**kw)
    assert rc != 0 and msg.startswith("wl_distill_update") and match in msg, msg


def test_distill_state_floats_and_workspace_queries_refuse_bad_sizes():
    import wheeledlab_b200 as wl
    assert wl.lib.wl_distill_state_floats(128, 3) == 4 + 384
    for T, E in ((0, 1), (8, 0)):
        assert wl.lib.wl_distill_state_floats(T, E) == 0 and b"wl_distill_state_floats" in wl.lib.wl_last_error()
    for D, N, G in ((0, 64, 15), (4097, 64, 15), (14, 0, 15), (14, 64, 0)):
        assert wl.lib.wl_distill_workspace_bytes(D, N, G) == 0 and b"wl_distill_workspace_bytes" in wl.lib.wl_last_error()


def test_fused_distillation_refuses_before_any_launch(monkeypatch):
    from wheeledlab_b200 import learner
    from wheeledlab_b200.learner import DistillationConfig, FusedDistillation
    s, _ = _blobs()
    monkeypatch.setattr(learner, "lib", _NoLaunch())
    with pytest.raises(NotImplementedError, match="loss_type='huber'"):
        FusedDistillation(s, 14, 32, 64, DistillationConfig(loss_type="huber"))
    with pytest.raises(ValueError, match="gradient_length 15"):
        FusedDistillation(s, 14, 8, 64, DistillationConfig())
    with pytest.raises(NotImplementedError, match="at most 16"):
        FusedDistillation(torch.zeros(100000), 17, 32, 64, DistillationConfig())
    with pytest.raises(ValueError, match="blob_layout\\(14\\)"):
        FusedDistillation(s[:-4], 14, 32, 64, DistillationConfig())


def test_the_run_scripts_distillation_agent_cfg_and_teacher_group():
    sys.path.insert(0, str(ROOT / "tools"))
    import ppo_train
    from wheeledlab_b200.learner import DistillationConfig, FusedOnPolicyRunner
    from wheeledlab_b200.runs import distillation_agent_cfg
    s = FusedOnPolicyRunner.settings(distillation_agent_cfg("relu", 64, 10))
    assert s.distillation and s.activation == "relu" and s.num_steps_per_env == 64 and s.alg_cfg == DistillationConfig()
    assert [fn for _, fn, _ in ppo_train.teacher_group("drift", None)] == ["root_pos_w", "root_euler_xyz", "base_lin_vel",
                                                                          "base_ang_vel", "last_action"]
    elev = ppo_train.teacher_group("elevation", None)
    assert elev[-1] == ("world_height_map", "world_height_map", {"clip": (-10.0, 10.0)})
    with pytest.raises(SystemExit, match="Drift family and Elevation"):
        ppo_train.teacher_group("visual", None)
