"""Distillation on the device (DESIGN 6t), against the fp64 restatement of rsl_rl's StudentTeacher + Distillation
(tests/distill_reference.py):
- the teacher row is the critic row of the same table, bit for bit, and the teacher's action is wl_actor_mean on it;
- one wl_distill_update at Drift obs 14 (ELU) and Elevation obs 689 (ReLU): the chunk gradient, blob, Adam moments and the
  per-step losses per element; the ReLU case on a margin batch (no layer-1 or layer-2 pre-activation within 1e-4 of 0);
- T % gradient_length != 0, several epochs (a chunk that wraps into the next epoch), max_grad_norm set and unset;
- the critic blocks, std and padding are never written, and two identical updates give identical bits;
- the captured DistillationIteration equals the eager one bit for bit;
- the runner distils a teacher the PPO runner trained: Loss/behavior follows the restatement over 3 iterations, the
  checkpoint round-trips, and the student plays through get_inference_policy."""
import pytest
import torch

from distill_reference import TorchDistillation

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
TEACHER = [("euler", "root_euler_xyz", {}), ("lin", "base_lin_vel", {}), ("ang", "base_ang_vel", {}),
           ("act", "last_action", {"clip": (-1.0, 1.0)}), ("mu", "wheel_friction", {})]              # 15 floats
ELEV_TEACHER = [("goal_relative_xyz", "goal_relative_xyz", {"clip": (-5.0, 5.0)}), ("root_euler_xyz", "root_euler_xyz", {}),
                ("base_lin_vel", "base_lin_vel", {"clip": (-10.0, 10.0)}), ("base_ang_vel", "base_ang_vel", {"clip": (-10.0, 10.0)}),
                ("last_action", "last_action", {"clip": (-1.0, 1.0)}),
                ("world_height_map", "world_height_map", {"clip": (-0.5, 0.5)}), ("mu", "wheel_friction", {})]   # 693 floats


def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")


def _bits(x):
    return x.contiguous().view(torch.int32)


def _drift_env(n, seed=4, teacher=None, critic=None):
    import wheeledlab_b200 as wl
    env = wl.ManagerBasedRLEnv(wl.make_task("Isaac-MushrDriftRL-v0", num_envs=n, seed=seed), device=DEV)
    if teacher:
        env.set_teacher_observation(teacher)
    if critic:
        env.set_critic_observation(critic)
    return env


def _student(D, act="elu", seed=0, std=(0.7, 1.3), critic=True):
    """A student blob: torch-initialised actor; the critic blocks random too (never stepped) unless critic=False."""
    from wheeledlab_b200.policy import pack_actor_critic
    torch.manual_seed(seed)
    a = torch.nn.ELU if act == "elu" else torch.nn.ReLU
    mk = lambda out: torch.nn.Sequential(torch.nn.Linear(D, 64), a(), torch.nn.Linear(64, 64), a(), torch.nn.Linear(64, out))
    crit = mk(1)
    if not critic:
        with torch.no_grad():
            for p in crit.parameters():
                p.zero_()
    return pack_actor_critic(mk(2), crit, torch.tensor(std), D, DEV)


def _params_mask(D):
    """(actor mask, any-parameter mask) over the blob."""
    from wheeledlab_b200.policy import actor_critic_state_dict, load_actor_critic_state_dict, blob_layout
    n = blob_layout(D)[1]
    marker = torch.arange(n, dtype=torch.float32, device=DEV) + 1
    touched = load_actor_critic_state_dict(actor_critic_state_dict(marker, D), D, out=torch.zeros_like(marker)) != 0
    o = blob_layout(D)[0]
    actor = torch.zeros_like(touched)
    actor[:o[6]] = touched[:o[6]]
    return actor, touched


def _margin_rows(blob, D, obs, act, margin=1e-4, rounds=8, seed=9):
    """Redraw every observation row whose fp64 layer-1 or layer-2 pre-activation (under `blob`'s actor) lies within `margin`
    of 0, so fp32 and fp64 take the same ReLU masks."""
    from wheeledlab_b200.policy import actor_critic_state_dict
    if act != "relu":
        return obs
    sd = {k: v.double() for k, v in actor_critic_state_dict(blob, D).items()}
    g = torch.Generator(device=DEV).manual_seed(seed)
    x = obs.reshape(-1, D)
    for _ in range(rounds):
        z1 = x.double() @ sd["actor.0.weight"].t() + sd["actor.0.bias"]
        z2 = torch.relu(z1) @ sd["actor.2.weight"].t() + sd["actor.2.bias"]
        bad = ((z1.abs() < margin).any(1)) | ((z2.abs() < margin).any(1))
        if not bool(bad.any()):
            return x.view_as(obs)
        x[bad] = 0.5 * torch.randn(int(bad.sum()), D, device=DEV, generator=g)
    raise AssertionError("no margin batch")


def _problem(D, act, T, N, seed=1):
    blob = _student(D, act, seed=seed)
    g = torch.Generator(device=DEV).manual_seed(100 + seed)
    obs = 0.5 * torch.randn(T, N, D, device=DEV, generator=g)
    obs = _margin_rows(blob, D, obs, act).contiguous()
    ta = 0.5 * torch.randn(T, N, 2, device=DEV, generator=g)
    return blob, obs, ta


def _grad_blob(ref_grads, D):
    """The restatement's student gradient (student order) in the blob layout."""
    from wheeledlab_b200.policy import blob_layout, load_actor_critic_state_dict
    names = [f"actor.{k}.{w}" for k in (0, 2, 4) for w in ("weight", "bias")]
    sd = {n: g.float() for n, g in zip(names, ref_grads)}
    sd["std"] = torch.zeros(2, device=DEV)
    return load_actor_critic_state_dict(sd, D, out=torch.zeros(blob_layout(D)[1], device=DEV), actor_only=True)


def _run(D, act, T, N, cfg, seed=1):
    from wheeledlab_b200.learner import FusedDistillation
    blob, obs, ta = _problem(D, act, T, N, seed)
    blob0 = blob.clone()
    alg = FusedDistillation(blob, D, T, N, cfg, act)
    alg.update(obs, ta)
    torch.cuda.synchronize()
    ref = TorchDistillation(blob0, D, cfg, act, dtype=torch.float64)
    ref_stats = ref.update(obs, ta)
    return blob0, alg, ref, ref_stats


def _check_update(D, act, alg, ref, ref_stats, cfg, T):
    from wheeledlab_b200.policy import actor_critic_state_dict, blob_layout
    E, G = cfg.num_learning_epochs, cfg.gradient_length
    n_steps = (E * T) // G
    assert float(alg.state[1]) == n_steps and float(alg.state[3]) == n_steps and len(ref.chunk_grads) == n_steps
    # the per-step losses (every one of the E * T, the unstepped tail included) and their mean
    got = alg.losses.double()
    want = torch.tensor(ref.losses, dtype=torch.float64, device=DEV)
    assert got.numel() == E * T and torch.allclose(got, want, rtol=2e-5, atol=1e-8), (got - want).abs().max()
    assert float(alg.state[2]) == pytest.approx(ref_stats["behavior"], rel=2e-5)
    # the last Adam step's reduced gradient (before clipping), per element
    o = blob_layout(D)[0]
    g = torch.zeros(blob_layout(D)[1], device=DEV)
    g[:o[6]] = alg.last_gradient()
    gref = _grad_blob(ref.chunk_grads[-1], D)
    actor, _ = _params_mask(D)
    gmax = gref[actor].abs().max()
    err = (g - gref).abs()
    assert bool((err[actor] <= 1e-5 * gmax + 1e-4 * gref[actor].abs()).all()), float((err[actor] / gmax).max())
    # the blob and the moments, per element: a step's error is the Adam ratio's, tiny where the gradient is well above the
    # rounding of its sum; entries whose gradient is within 1e-3 of the largest get half a step of room
    sd_got, sd_ref = actor_critic_state_dict(alg.blob, D), ref.state_dict()
    m_ref = ref.adam_moments()
    m_got, v_got = actor_critic_state_dict(alg.m, D), actor_critic_state_dict(alg.v, D)
    gsd = actor_critic_state_dict(gref, D)
    for name, w in sd_ref.items():
        step = cfg.learning_rate * n_steps
        small = gsd[name].abs() < 1e-3 * gmax
        tol = torch.where(small, 0.5 * step, 1e-3 * step) + 1e-7
        assert bool(((sd_got[name].double() - w).abs() <= tol).all()), (name, float((sd_got[name].double() - w).abs().max()))
        mr, vr = m_ref[name]
        assert torch.allclose(m_got[name].double(), mr, atol=1e-4 * float(mr.abs().max()), rtol=0), name
        assert torch.allclose(v_got[name].double(), vr, atol=1e-4 * float(vr.abs().max()), rtol=0), name


CASES = [  # (obs_dim, activation, T, N, epochs, gradient_length, max_grad_norm)
    (14, "elu", 30, 256, 1, 15, None),
    (14, "elu", 30, 256, 1, 15, 1.0),
    (689, "relu", 15, 128, 1, 15, None),
    (689, "relu", 15, 128, 1, 15, 0.05),
    (14, "elu", 20, 128, 1, 15, None),           # T % G: the last 5 steps are evaluated, not stepped
    (14, "elu", 20, 128, 3, 15, 0.05),           # epochs: chunks [15, 30) and [45, 60) wrap into the next epoch; clipped
    (14, "elu", 16, 100, 2, 3, None),            # N not a multiple of the 64-sample tile, a 2-step tail
]


@pytest.mark.parametrize("D,act,T,N,E,G,mgn", CASES, ids=[f"D{c[0]}-{c[1]}-T{c[2]}-N{c[3]}-E{c[4]}-G{c[5]}-clip{c[6]}" for c in CASES])
def test_update_matches_the_fp64_restatement(D, act, T, N, E, G, mgn):
    _need_gpu()
    from wheeledlab_b200.learner import DistillationConfig
    cfg = DistillationConfig(num_learning_epochs=E, gradient_length=G, learning_rate=1e-3, max_grad_norm=mgn)
    _, alg, ref, ref_stats = _run(D, act, T, N, cfg)
    _check_update(D, act, alg, ref, ref_stats, cfg, T)


@pytest.mark.parametrize("D,act", [(14, "elu"), (689, "relu")])
def test_update_steps_the_actor_alone_and_repeats_bit_for_bit(D, act):
    _need_gpu()
    from wheeledlab_b200.learner import DistillationConfig, FusedDistillation
    cfg = DistillationConfig(num_learning_epochs=2, gradient_length=5, max_grad_norm=1.0)
    T, N = 12, 96
    blob, obs, ta = _problem(D, act, T, N, seed=3)
    actor, params = _params_mask(D)
    runs = []
    for _ in range(2):
        b = blob.clone()
        alg = FusedDistillation(b, D, T, N, cfg, act)
        alg.update(obs, ta)
        runs.append(alg)
    torch.cuda.synchronize()
    a, b = runs
    for x, y in ((a.blob, b.blob), (a.m, b.m), (a.v, b.v), (a.state, b.state), (a.last_gradient(), b.last_gradient())):
        assert torch.equal(_bits(x), _bits(y))
    assert torch.equal(_bits(a.blob[~actor]), _bits(blob[~actor])), "a critic, std or padding float was written"
    assert bool((a.m[~actor] == 0).all()) and bool((a.v[~actor] == 0).all())
    assert bool((a.blob[actor] != blob[actor]).float().mean() > 0.9)
    assert bool((blob[~params] == 0).all())


def test_teacher_row_is_the_critic_row_and_the_teacher_action_is_actor_mean():
    _need_gpu()
    import wheeledlab_b200 as wl
    from wheeledlab_b200.learner import DistillationConfig, DistillationIteration
    from wheeledlab_b200.policy import actor_mean
    a, b = _drift_env(64, teacher=TEACHER), _drift_env(64, critic=TEACHER)
    assert a.observation_manager.group_obs_dim["teacher"] == (15,) and "critic" not in a.observation_manager.group_obs_dim
    _, ea = a.reset()
    _, eb = b.reset()
    assert torch.equal(_bits(ea["observations"]["teacher"]), _bits(eb["observations"]["critic"]))
    for t in range(4):
        act = a.sim.synth_actions(t)
        ea, eb = a.step(act)[4], b.step(act)[4]
        assert set(ea["observations"]) == {"policy", "teacher"}
        assert torch.equal(_bits(ea["observations"]["teacher"]), _bits(eb["observations"]["critic"]))
    assert torch.equal(_bits(a.get_observations()[1]["observations"]["teacher"]), _bits(b.sim.critic_observe()))
    with pytest.raises(NotImplementedError, match="not both"):
        a.set_critic_observation(TEACHER)
    with pytest.raises(NotImplementedError, match="not both"):
        b.set_teacher_observation(TEACHER)
    with pytest.raises(NotImplementedError, match="Visual"):
        wl.make("Isaac-MushrVisualRL-v0", device=DEV, num_envs=8, seed=1).set_teacher_observation(TEACHER)
    # the iteration's teacher action of each step is wl_actor_mean on the teacher row the step starts from
    for env, D, Dt, act in ((a, 14, 15, "elu"), (_elev_env(64), 689, 693, "relu")):
        it = DistillationIteration(env.sim, _student(D, act, critic=False), _student(Dt, act, seed=5, critic=False),
                                   DistillationConfig(gradient_length=4), T=8, activation=act)
        it.start(env.common_step_counter, capture=False)
        rows = []
        sim_critic = env.sim.critic_observe
        it.sim.critic_observe = lambda out=None: (sim_critic(out=out), rows.append(out.clone()))[0]
        t0 = it.tobs.clone()
        it.run()
        del it.sim.critic_observe
        torch.cuda.synchronize()
        for k, row in enumerate([t0] + rows[:-1]):
            assert torch.equal(_bits(it.slab.teacher_actions[k]), _bits(actor_mean(it.teacher_blob, Dt, row, act))), (D, k)
        assert bool(torch.isfinite(it.alg.losses).all()) and float(it.alg.state[1]) == 2


def _elev_env(n, seed=11):
    import wheeledlab_b200 as wl
    env = wl.ManagerBasedRLEnv(wl.elevation_task(num_envs=n, seed=seed), device=DEV)
    env.set_teacher_observation(ELEV_TEACHER)
    return env


@pytest.mark.parametrize("task", ["drift", "elevation"])
def test_captured_iteration_equals_the_eager_one(task):
    _need_gpu()
    from wheeledlab_b200.learner import DistillationConfig, DistillationIteration
    D, Dt, act = (14, 15, "elu") if task == "drift" else (689, 693, "relu")
    outs, chained = [], []
    for capture in (False, True):
        env = _drift_env(256, teacher=TEACHER) if task == "drift" else _elev_env(128)
        env.reset()
        it = DistillationIteration(env.sim, _student(D, act, critic=False), _student(Dt, act, seed=5, critic=False),
                                   DistillationConfig(num_learning_epochs=2, gradient_length=6, max_grad_norm=1.0), T=16, activation=act)
        it.start(env.common_step_counter, capture=capture)
        for _ in range(2):
            it.run()
        torch.cuda.synchronize()
        assert (it.graph is not None) == capture
        outs.append({"blob": it.blob, "m": it.alg.m, "v": it.alg.v, "state": it.alg.state, "slab": it.slab.flat,
                     "teacher_actions": it.slab.teacher_actions, "readback": it.readback, "tobs": it.tobs})
        chained.append(env.sim.chained_step_count)
    differ = [k for k in outs[0] if not torch.equal(outs[0][k].view(torch.uint8), outs[1][k].view(torch.uint8))]
    assert not differ, (differ, "chained steps (eager, captured)", chained)


def _ppo_cfg(T):
    from dataclasses import asdict
    from wheeledlab_b200.learner import PPOConfig
    return {"num_steps_per_env": T, "save_interval": 100, "empirical_normalization": False,
            "policy": {"class_name": "ActorCritic", "init_noise_std": 1.0, "actor_hidden_dims": [64, 64], "critic_hidden_dims": [64, 64],
                       "activation": "elu"},
            "algorithm": {"class_name": "PPO", **asdict(PPOConfig())}}


def _distill_cfg(T, E=2, G=8):
    return {"num_steps_per_env": T, "save_interval": 1, "empirical_normalization": False,
            "policy": {"class_name": "StudentTeacher", "init_noise_std": 0.5, "noise_std_type": "scalar", "student_hidden_dims": [64, 64],
                       "teacher_hidden_dims": [64, 64], "activation": "elu"},
            "algorithm": {"class_name": "Distillation", "num_learning_epochs": E, "gradient_length": G, "learning_rate": 1e-3,
                          "max_grad_norm": 1.0, "loss_type": "mse"}}


def test_runner_distils_a_ppo_teacher_saves_loads_and_plays(tmp_path):
    _need_gpu()
    from wheeledlab_b200.learner import DistillationIteration, FusedOnPolicyRunner
    from wheeledlab_b200.policy import actor_critic_state_dict, actor_mean, student_teacher_state_dict
    # the teacher: PPO on an env whose policy row is the teacher row
    env_p = _drift_env(512)
    env_p.set_policy_observation(TEACHER)
    torch.manual_seed(3)
    rp = FusedOnPolicyRunner(env_p, _ppo_cfg(24), device=DEV)
    rp.learn(2)
    rp.save(str(tmp_path / "teacher.pt"))
    # the student
    env = _drift_env(512, teacher=TEACHER)
    torch.manual_seed(4)
    cfg = _distill_cfg(24)
    r = FusedOnPolicyRunner(env, cfg, log_dir=str(tmp_path / "run"), device=DEV)
    assert type(r.it) is DistillationIteration and r.distillation
    with pytest.raises(ValueError, match="Teacher model parameters not loaded"):
        r.learn(1)
    r.load(str(tmp_path / "teacher.pt"))
    assert r.current_learning_iteration == 0 and float(r.alg.state[1]) == 0
    want = actor_critic_state_dict(rp.blob, 15)
    got = student_teacher_state_dict(r.blob, 14, r.teacher_blob, 15)
    assert all(torch.equal(got[f"teacher.{k}.{w}"], want[f"actor.{k}.{w}"]) for k in (0, 2, 4) for w in ("weight", "bias"))
    from wheeledlab_b200.learner import DistillationConfig
    ref = TorchDistillation(r.blob.clone(), 14, DistillationConfig.from_rsl_rl(type("A", (), cfg["algorithm"])), "elu")
    logs, slabs = [], []
    r.callback = lambda k, log: (logs.append(log), slabs.append((r.it.slab.obs_in.clone(), r.it.slab.teacher_actions.clone())))
    r.learn(3)
    assert r.it.graph is not None and len(logs) == 3
    for log, (obs, ta) in zip(logs, slabs):
        assert log["Loss/behavior"] == pytest.approx(ref.update(obs, ta)["behavior"], rel=1e-4)
        assert log["Loss/learning_rate"] == pytest.approx(1e-3) and log["Policy/mean_noise_std"] == pytest.approx(0.5)
        assert "Perf/total_fps" in log and "Episodes/finished" in log
    assert logs[-1]["Loss/behavior"] < logs[0]["Loss/behavior"]
    assert (tmp_path / "run" / "models" / "model_2.pt").exists()
    # save, load into a fresh runner: everything resumes
    r.save(str(tmp_path / "st.pt"))
    d = torch.load(str(tmp_path / "st.pt"), map_location=DEV)
    assert sorted(d["model_state_dict"]) == sorted(got) and list(d["optimizer_state_dict"]["state"]) == list(range(6))
    r2 = FusedOnPolicyRunner(_drift_env(512, seed=9, teacher=TEACHER), cfg, device=DEV)
    r2.load(str(tmp_path / "st.pt"))
    for x, y in ((r.blob, r2.blob), (r.teacher_blob, r2.teacher_blob), (r.alg.m, r2.alg.m), (r.alg.v, r2.alg.v)):
        assert torch.equal(_bits(x), _bits(y))
    assert r2.current_learning_iteration == 2 and float(r2.alg.state[1]) == float(r.alg.state[1])
    log = r2.learn(1)
    assert r2.current_learning_iteration == 2 and float(r2.alg.state[1]) == float(r.alg.state[1]) + 6 and log["Loss/behavior"] > 0
    # the student plays
    policy = r.get_inference_policy()
    obs, _ = env.get_observations()
    a = policy(obs)
    assert torch.equal(_bits(a), _bits(actor_mean(r.blob, 14, obs, "elu")))
    env.step(a)


def test_ppo_train_distils_a_checkpoint_and_play_policy_plays_the_student(tmp_path):
    _need_gpu()
    import subprocess
    import sys
    from pathlib import Path
    root = Path(__file__).resolve().parent.parent
    sys.path.insert(0, str(root / "tools"))
    import play_policy
    run = lambda *args: subprocess.run([sys.executable, str(root / "tools" / "ppo_train.py"), "--envs", "256", "--steps", "16",
                                        "--save-interval", "1", *args], capture_output=True, text=True, check=True).stdout
    run("--iters", "2", "--log-dir", str(tmp_path / "ppo"))
    out = run("--iters", "2", "--log-dir", str(tmp_path / "dist"), "--teacher", str(tmp_path / "ppo" / "models" / "model_1.pt"))
    assert "distillation of model_1.pt (teacher row 14)" in out and "behavior" in out
    ck = torch.load(str(tmp_path / "dist" / "models" / "model_1.pt"), map_location="cpu")
    assert "student.0.weight" in ck["model_state_dict"] and ck["iter"] == 1
    args = play_policy.parser().parse_args(["-p", str(tmp_path / "dist"), "--steps", "20"])
    r = play_policy.resolve(args)
    assert r["teacher_terms"] and r["agent_cfg"]["policy"]["class_name"] == "StudentTeacher"
    runner, roll, _ = play_policy.play(r, 20)
    from wheeledlab_b200.policy import student_teacher_state_dict
    got = student_teacher_state_dict(runner.blob, 14, runner.teacher_blob, 14)
    assert all(torch.equal(got[k].cpu(), v) for k, v in ck["model_state_dict"].items())
    assert roll.slab.actions.shape == (20, 256, 2) and bool(torch.isfinite(roll.slab.actions).all())
