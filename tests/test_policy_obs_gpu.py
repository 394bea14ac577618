"""A modified policy observation group on the device (wl_policy_observe, DESIGN 6q):
- the kernel equals the CPU twin bit for bit at several sizes, on host and device counters, for dropped and reordered terms,
  every noise kind, clips and scales, rows of 1 to 32 floats, and output rows that are not 16-byte aligned;
- BlindObsCfg's five terms forced through a table equal the built-in row over 1000 steps with resets, with and without
  enable_corruption, on Drift and F1Tenth, after steps and for observe calls (env.reset / get_observations);
- a captured graph of device-counter steps replays to the rows of the eager host-counter steps;
- the env returns the table's row; the fused entries refuse a handle with a table;
- the runner trains on the table's row in one graph (alone, with a critic group, with a device reward term and push),
  resumes bit for bit, refuses a checkpoint of another width, keeps data-parallel replicas equal, and plays back."""
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent))

pytestmark = pytest.mark.gpu

if not torch.cuda.is_available():
    pytest.skip("needs a CUDA device", allow_module_level=True)

import wheeledlab_b200 as wl                                   # noqa: E402
from wheeledlab_b200 import policy_obs                         # noqa: E402
from wheeledlab_b200.env import ManagerBasedRLEnv              # noqa: E402
from wheeledlab_b200.sim import WheeledSim                     # noqa: E402
from oracle_lib import policy_observe                           # noqa: E402

DEV = "cuda:0"
NO_POS = [("root_euler_xyz", ("gaussian", 0.0, 0.1), None, None), ("base_lin_vel", ("gaussian", 0.0, 0.5), None, None),
          ("base_ang_vel", ("gaussian", 0.0, 0.4), None, None), ("last_action", None, (-1.0, 1.0), None)]            # 11 floats
TABLES = {
    "dp1": [("base_mass", ("uniform", -0.5, 0.25), None, 2.0)],
    "dp11_dropped": NO_POS,
    "dp11_reordered": [NO_POS[3], NO_POS[1], NO_POS[0], NO_POS[2]],
    "dp16": [("projected_gravity", ("gaussian", 0.3, 0.05), (-0.9, 0.8), None), ("base_lin_vel", ("uniform", -0.5, 0.5), None, (1.0, 2.0, 3.0)),
             ("joint_vel", ("gaussian", 0.0, 0.2), (-30.0, 10.0), 0.05), ("joint_pos", None, None, (4.0, -4.0)),
             ("last_action", ("uniform", 0.0, 0.1), (-1.0, 1.0), None), ("root_pos_w", ("gaussian", -0.2, 0.1), None, None)],
    "dp17": [("wheel_friction", ("gaussian", 0.0, 0.1), None, None), ("motor_damping", ("uniform", -1.0, 1.0), (-0.5, 0.5), 3.0),
             ("base_mass", None, None, None), ("root_euler_xyz", ("gaussian", 0.0, 0.1), None, (0.5, 0.5, 0.25)),
             ("base_ang_vel", ("uniform", -0.4, 0.4), None, None), ("last_action", None, (-0.5, 1.0), None)],
    "dp32": [("projected_gravity", ("gaussian", 0.0, 0.05), None, None), ("base_ang_vel", ("gaussian", 0.0, 0.4), None, None),
                  ("base_lin_vel", ("uniform", -0.5, 0.5), None, None), ("last_action", None, (-1.0, 1.0), None),
                  ("joint_vel", ("gaussian", 0.1, 0.2), None, 0.01), ("joint_pos", ("uniform", 0.0, 0.1), (-0.3, 0.2), None),
                  ("wheel_friction", ("gaussian", 0.0, 0.1), None, None), ("base_mass", ("uniform", -1.0, 1.0), None, 0.5),
                  ("motor_damping", None, (-0.5, 0.5), (1.0, 2.0, 3.0, 4.0)), ("root_euler_xyz", ("gaussian", 0.0, 0.1), None, None),
                  ("root_pos_w", None, None, None)],
}


def _sim(task, n, seed=11, offset=0, corrupt=None):
    spec = wl.make_task(task, num_envs=n, seed=seed, env_id_offset=offset)
    if corrupt is not None:
        spec.cfg.enable_corruption = int(corrupt)
    sim = WheeledSim(spec, DEV)
    sim.startup()
    sim.reset(None, 0)
    return sim


def _bits(x):
    return x.contiguous().view(torch.int32).cpu().numpy()


def _twin(sim, table, t, call_idx=-1):
    c = sim.cfg
    return policy_observe(int(c.seed), int(c.env_id_offset), sim.groups.cpu().numpy(), table, bool(c.enable_corruption), t, call_idx)


def _run(sim, steps, t0=0):
    for t in range(t0, t0 + steps):
        sim.step(sim.synth_actions(t), t)


# ---- 1. the kernel against the twin ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [1, 33, 4096, 8192])
@pytest.mark.parametrize("table", sorted(TABLES))
def test_kernel_equals_the_twin(n, table):
    sim = _sim("drift", n, offset=7)
    _run(sim, 40)
    dp = sim.set_policy_terms(TABLES[table])
    assert dp == policy_obs.row_width(TABLES[table]) == sim.policy_obs_dim and sim.obs_dim == 14
    torch.cuda.synchronize()
    for call_idx in (-1, 0, 3):
        want = _twin(sim, TABLES[table], 39, call_idx)
        got = sim.policy_observe(39, None if call_idx < 0 else call_idx)
        assert np.array_equal(_bits(got), want.view(np.int32)), (table, n, call_idx)
        # an output row that is not 16-byte aligned (a slab row of an odd N * Dp)
        buf = torch.full((n * dp + 1,), float("nan"), device=DEV)
        sim.policy_observe(39, None if call_idx < 0 else call_idx, out=buf[1:].view(n, dp))
        assert np.array_equal(_bits(buf[1:].view(n, dp)), want.view(np.int32)) and torch.isnan(buf[0])
    sim.set_step_counter(30)                                   # WL_DEVICE_COUNTER_PLUS(9) = 30 + 9
    got = sim.policy_observe(WheeledSim.device_counter_plus(9))
    assert np.array_equal(_bits(got), _twin(sim, TABLES[table], 39).view(np.int32))


def test_two_shards_equal_one_handle():
    table = TABLES["dp32"]
    whole = _sim("drift", 256)
    halves = [_sim("drift", 128, offset=0), _sim("drift", 128, offset=128)]
    halves[0].groups.copy_(whole.groups[:, :128])
    halves[1].groups.copy_(whole.groups[:, 128:])
    for s in [whole] + halves:
        s.set_policy_terms(table)
    got = torch.cat([h.policy_observe(5) for h in halves])
    assert torch.equal(got.view(torch.int32), whole.policy_observe(5).view(torch.int32))


# ---- 2. BlindObsCfg through a table is the built-in row ---------------------------------------------------------------------
@pytest.mark.parametrize("task", ["drift", "f1tenth_drift"])
@pytest.mark.parametrize("corrupt", [True, False])
def test_the_blind_group_through_a_table_is_the_built_in_row(task, corrupt):
    sim = _sim(task, 512, corrupt=corrupt)
    sim.set_policy_terms(policy_obs.blind_table(list(sim.cfg.noise_std)))
    resets = 0
    for t in range(1000):
        obs, _, term, trunc = sim.step(sim.synth_actions(t), t)
        resets += int((term | trunc).sum())
        # equal as fp32 values: a -0 that the built-in row's "+ std * z" turns into +0 may stay -0 without noise
        assert torch.equal(sim.policy_observe(t), obs), f"step {t}"
        if t % 97 == 0:
            for ci in (0, 1, 7):
                assert torch.equal(sim.policy_observe(t + 1, ci), sim.observe(t + 1, ci)), f"observe {t} {ci}"
    assert resets > 0


def test_env_with_the_blind_table_returns_the_built_in_rows():
    a = ManagerBasedRLEnv(wl.make_task("drift", num_envs=256, seed=3), device=DEV)
    b = ManagerBasedRLEnv(wl.make_task("drift", num_envs=256, seed=3), device=DEV)
    b.set_policy_observation([(n, fn, {"noise": nz, "clip": cl}) for n, (fn, nz, cl, _) in
                              zip("abcde", policy_obs.blind_table(list(b.sim.cfg.noise_std)))])
    assert b.observation_manager.group_obs_dim["policy"] == (14,)
    for x, y in ((a.reset()[0]["policy"], b.reset()[0]["policy"]), (a.get_observations()[0], b.get_observations()[0])):
        assert torch.equal(x, y)
    for t in range(50):
        act = a.sim.synth_actions(t)
        assert torch.equal(a.step(act)[0]["policy"], b.step(act)[0]["policy"]), t
    assert torch.equal(a.get_observations()[0], b.get_observations()[0])


# ---- 3. graph capture -------------------------------------------------------------------------------------------------------
def test_captured_device_counter_graph_equals_eager_host_counters():
    n, K, R, table = 512, 4, 3, TABLES["dp17"]
    a, b = _sim("drift", n), _sim("drift", n)
    for s in (a, b):
        s.set_policy_terms(table)
    gen = torch.Generator(device=DEV).manual_seed(9)
    acts = [torch.rand((n, 2), device=DEV, generator=gen) * 2 - 1 for _ in range(K * R)]
    ref = []
    for t in range(K * R):
        a.step(acts[t], t)
        ref.append(a.policy_observe(t).clone())
    scratch = [(torch.empty((n, 14), device=DEV), torch.empty(n, device=DEV), torch.empty(n, dtype=torch.uint8, device=DEV),
                torch.empty(n, dtype=torch.uint8, device=DEV)) for _ in range(K)]
    outs = [torch.empty_like(ref[0]) for _ in range(K)]
    acts_k = [torch.empty_like(acts[0]) for _ in range(K)]
    stream = torch.cuda.Stream()
    stream.wait_stream(torch.cuda.current_stream())
    g = torch.cuda.CUDAGraph()
    b.set_step_counter(0)
    with torch.cuda.stream(stream), torch.cuda.graph(g, stream=stream):
        for k in range(K):
            b.step(acts_k[k], WheeledSim.device_counter_plus(k), out=scratch[k])
            b.policy_observe(WheeledSim.device_counter_plus(k), out=outs[k])
        b.advance_counter(K)
    torch.cuda.current_stream().wait_stream(stream)
    b.set_step_counter(0)
    for r in range(R):
        for k in range(K):
            acts_k[k].copy_(acts[r * K + k])
        g.replay()
        torch.cuda.synchronize()
        for k in range(K):
            assert torch.equal(ref[r * K + k].view(torch.int32), outs[k].view(torch.int32)), f"replay {r} step {k}"


# ---- 4. the env, and what refuses a table -----------------------------------------------------------------------------------
def test_env_returns_the_tables_row_after_step_reset_and_get_observations():
    env = ManagerBasedRLEnv(wl.make_task("drift", num_envs=300, seed=5), device=DEV)
    env.set_policy_observation([(f"t{k}", fn, {"noise": nz, "clip": cl, "scale": sc}) for k, (fn, nz, cl, sc) in enumerate(TABLES["dp11_dropped"])])
    assert env.observation_manager.group_obs_dim["policy"] == (11,) and env.observation_space["policy"].shape == (300, 11)
    obs, _ = env.reset()
    assert np.array_equal(_bits(obs["policy"]), _twin(env.sim, NO_POS, 0, 0).view(np.int32))
    for t in range(30):
        obs, *_ = env.step(env.sim.synth_actions(t))
        assert obs["policy"].shape == (300, 11)
        assert np.array_equal(_bits(obs["policy"]), _twin(env.sim, NO_POS, t).view(np.int32)), t
    o, extras = env.get_observations()
    assert np.array_equal(_bits(o), _twin(env.sim, NO_POS, 30, 1).view(np.int32))        # reset() was observe call 0
    env.set_policy_observation([])
    assert env.observation_manager.group_obs_dim["policy"] == (14,) and env.step(env.sim.synth_actions(30))[0]["policy"].shape == (300, 14)


@pytest.mark.parametrize("other", ["critic", "device_term"])
def test_env_table_with_a_critic_group_or_a_device_reward_term(other):
    from wheeledlab_b200 import device_terms as dtm, privileged
    env = ManagerBasedRLEnv(wl.make_task("drift", num_envs=128, seed=6), device=DEV)
    if other == "critic":
        env.set_critic_observation([("friction", privileged.wheel_friction), ("vel", "base_lin_vel")])
    else:
        env.add_device_reward_term("fv", dtm.resolve("forward_vel", "wheeledlab_tasks.elevation.mushr_elevation_env_cfg"), 1.0)
    table = [("projected_gravity", ("gaussian", 0.0, 0.05), None, None), ("joint_vel", ("uniform", -0.1, 0.1), None, None)]
    env.set_policy_observation([("grav", "projected_gravity", {"noise": ("gaussian", 0.0, 0.05)}), ("spin", "joint_vel", {"noise": ("uniform", -0.1, 0.1)})])
    env.reset()
    for t in range(10):
        obs, *_ = env.step(env.sim.synth_actions(t))
        assert np.array_equal(_bits(obs["policy"]), _twin(env.sim, table, t).view(np.int32))
        if other == "critic":
            assert obs["critic"].shape == (128, 7)


def test_the_fused_entries_the_staged_step_and_the_runner_refuse_a_table():
    import ctypes as C
    from wheeledlab_b200._lib import WlPolicyOut, lib
    sim = _sim("drift", 64)
    sim.set_policy_terms(NO_POS)
    p = lambda x: C.c_void_p(x.data_ptr())
    obs, blob = torch.zeros((64, 14), device=DEV), torch.zeros(8192, device=DEV)
    f, u = torch.zeros(64 * 4, device=DEV), torch.zeros(64, dtype=torch.uint8, device=DEV)
    out = WlPolicyOut(p(f), p(f), p(f), p(f))
    assert lib.wl_act_step(sim._h, p(obs), p(blob), out, p(obs), p(f), p(u), p(u), None, 0, None) == -3
    assert b"policy observation table" in lib.wl_last_error()
    assert lib.wl_act_infer_step(sim._h, p(obs), p(blob), p(f), p(obs), p(f), p(u), p(u), None, 0, None) == -3
    assert b"policy observation table" in lib.wl_last_error()
    assert lib.wl_rollout(sim._h, 2, None, None, p(obs), p(f), p(u), p(u), p(f), 0, None) == -3
    assert b"policy observation table" in lib.wl_last_error()
    sim.step(sim.synth_actions(0), 0)                          # wl_step still writes the built-in row
    for bad in ([("lidar", None, None, None)], [("base_mass", ("gaussian", 0.0, float("nan")), None, None)],
                [("joint_vel", None, None, (1.0, 2.0))], NO_POS * 3):
        with pytest.raises((RuntimeError, ValueError)):
            sim.set_policy_terms(bad)
    assert sim.policy_obs_dim == 11, "a refused table leaves the handle's table as it was"
    with pytest.raises(ValueError, match="out must be"):
        sim.policy_observe(0, out=torch.empty((64, 14), device=DEV))
    elev = _sim("elevation", 16)
    with pytest.raises(RuntimeError, match="Drift family"):
        elev.set_policy_terms(NO_POS)
    env = ManagerBasedRLEnv(wl.make_task("drift", num_envs=64, seed=1), device=DEV)
    env.set_policy_observation([("yaw", "root_euler_xyz")])
    with pytest.raises(NotImplementedError, match="host-side Python"):
        env.add_reward_term("r", lambda e: e.sim.root_pos_w[:, 0], 1.0)
    from wheeledlab_b200.learner import FusedOnPolicyRunner
    from wheeledlab_b200.runs import agent_cfg
    wide = ManagerBasedRLEnv(wl.make_task("drift", num_envs=64, seed=1), device=DEV)
    wide.set_policy_observation([("spin", "joint_vel"), ("friction", "wheel_friction"), ("damping", "motor_damping"),
                                 ("mass", "base_mass"), ("steer", "joint_pos"), ("grav", "projected_gravity")])  # 18 floats
    with pytest.raises(NotImplementedError, match="at most 16 floats"):
        FusedOnPolicyRunner(wide, agent_cfg("elu", steps=8), device=DEV)
    FusedOnPolicyRunner(wide, agent_cfg("relu", steps=8), device=DEV).learn(1)     # the ReLU network takes it


# ---- 5. training and playback at the table's width -------------------------------------------------------------------------
T = 8
NO_POS_ENV = [(f"t{k}", fn, {"noise": nz, "clip": cl}) for k, (fn, nz, cl, _) in enumerate(NO_POS)]
PUSH = {"velocity_range": {"x": (-0.5, 0.5), "y": (-0.5, 0.5), "yaw": (-1.0, 1.0)}}


def _env(n=256, offset=0, extra=None):
    env = ManagerBasedRLEnv(wl.make_task("drift", num_envs=n, seed=4, env_id_offset=offset), device=DEV)
    if extra == "critic":
        from wheeledlab_b200 import privileged
        env.set_critic_observation([("friction", privileged.wheel_friction), ("vel", "base_lin_vel")])
    elif extra == "device":
        from wheeledlab_b200 import device_terms as dtm
        root = Path(__file__).resolve().parent.parent
        if str(root / "shims") not in sys.path:
            sys.path.insert(0, str(root / "shims"))
        from isaaclab.envs import mdp
        env.add_device_reward_term("fv", dtm.resolve("forward_vel", dtm.ELEVATION), 0.5)
        env.add_device_event_term("push", mdp.push_by_setting_velocity, "interval", (0.05, 0.2), PUSH)
    env.set_policy_observation(NO_POS_ENV)
    return env


def _runner(env, **kw):
    from wheeledlab_b200.learner import FusedOnPolicyRunner
    from wheeledlab_b200.runs import agent_cfg
    torch.manual_seed(0)
    return FusedOnPolicyRunner(env, agent_cfg("elu", steps=T, save_interval=1), device=DEV, **kw)


@pytest.mark.parametrize("extra", [None, "critic", "device"])
def test_runner_trains_on_the_table_in_one_graph_and_resumes_bit_for_bit(tmp_path, extra):
    from wheeledlab_b200.policy import actor_critic_state_dict
    env_a, env_b = _env(extra=extra), _env(extra=extra)
    a, b = _runner(env_a, log_dir=str(tmp_path)), _runner(env_b)
    assert a.it.roll.table and a.it.roll.slab.obs_in.shape[-1] == 11
    for r in (a, b):
        torch.manual_seed(21)
        r.learn(2)
    assert a.it.graph is not None and env_a.common_step_counter == 2 * T
    sd = actor_critic_state_dict(a.blob, 11, a.critic_obs_dim)
    assert tuple(sd["actor.0.weight"].shape) == (64, 11)
    assert tuple(sd["critic.0.weight"].shape) == ((64, 7) if extra == "critic" else (64, 11))
    c = _runner(env_b)
    c.load(str(tmp_path / "models" / "model_1.pt"))
    a.alg.state[0] = c.alg.cfg.learning_rate
    for r in (a, c):
        torch.manual_seed(22)
        r.learn(1)
    torch.cuda.synchronize()
    for name, x, y in (("blob", a.blob, c.blob), ("m", a.alg.m, c.alg.m), ("v", a.alg.v, c.alg.v)):
        assert np.array_equal(_bits(x), _bits(y)), name
    assert torch.equal(env_a.sim.groups, env_b.sim.groups)


def test_a_checkpoint_of_another_width_is_refused_with_the_blob_untouched(tmp_path):
    from wheeledlab_b200.learner import FusedOnPolicyRunner
    from wheeledlab_b200.runs import agent_cfg
    plain = ManagerBasedRLEnv(wl.make_task("drift", num_envs=64, seed=4), device=DEV)
    p = FusedOnPolicyRunner(plain, agent_cfg("elu", steps=T), device=DEV)
    p.save(str(tmp_path / "w14.pt"))
    r = _runner(_env(64))
    before = r.blob.clone()
    with pytest.raises(ValueError):
        r.load(str(tmp_path / "w14.pt"))
    assert np.array_equal(_bits(before), _bits(r.blob))


def test_the_rollout_graph_equals_eager_steps_on_the_table():
    """The captured rollout (policy kernel, step, wl_policy_observe into the next slab row) against the same calls made eagerly
    on host counters, in that order."""
    from wheeledlab_b200.policy import FusedPolicyRollout, pack_actor_critic, policy_act
    n = 512
    a, b = _sim("drift", n), _sim("drift", n)
    for s in (a, b):
        s.set_policy_terms(NO_POS)
    mk = lambda out: torch.nn.Sequential(torch.nn.Linear(11, 64), torch.nn.ELU(), torch.nn.Linear(64, 64), torch.nn.ELU(), torch.nn.Linear(64, out))
    torch.manual_seed(3)
    blob = pack_actor_critic(mk(2), mk(1), torch.full((2,), 1.0), 11, DEV)
    roll = FusedPolicyRollout(a, blob, T).capture(0)
    slab = roll.run()
    obs = b.policy_observe(0, 0)
    act, mean, lp, val = (torch.empty((n, 2), device=DEV), torch.empty((n, 2), device=DEV), torch.empty(n, device=DEV),
                          torch.empty(n, device=DEV))
    for t in range(T):
        assert torch.equal(obs.view(torch.int32), slab.obs_in[t].view(torch.int32)), t
        policy_act(b, obs, blob, act, mean, lp, val, t, "elu")
        assert torch.equal(act, slab.actions[t]) and torch.equal(val, slab.values[t])
        b.step(act, t)
        obs = b.policy_observe(t).clone()
    assert torch.equal(obs.view(torch.int32), roll.obs0.view(torch.int32))


def test_one_process_data_parallel_iteration_keeps_replicas_equal():
    from wheeledlab_b200.learner import LocalRanksIteration, PPOConfig, PPOExchange, PPOIteration
    from wheeledlab_b200.policy import pack_actor_critic
    R, n, D = 2, 512, 11
    mk = lambda out: torch.nn.Sequential(torch.nn.Linear(D, 64), torch.nn.ELU(), torch.nn.Linear(64, 64), torch.nn.ELU(), torch.nn.Linear(64, out))
    torch.manual_seed(7)
    blob = pack_actor_critic(mk(2), mk(1), torch.full((2,), 1.0), D, DEV)
    its = []
    for r, ex in enumerate(PPOExchange.local(R, D, DEV)):
        e = _env(n, offset=r * n); e.reset()
        its.append(PPOIteration(e.sim, blob.clone(), PPOConfig(), T, "elu", episode_stats=True, exchange=ex))
    group = LocalRanksIteration(its).start(0, capture=True)
    g = torch.Generator(device=DEV).manual_seed(1)
    for k in range(3):
        group.run([torch.randperm(n * T, device=DEV, generator=g) for _ in range(R)])
        torch.cuda.synchronize()
        a, b = group.its
        for x, y in ((a.blob, b.blob), (a.ppo.m, b.ppo.m), (a.ppo.v, b.ppo.v)):
            assert np.array_equal(_bits(x), _bits(y)), f"iteration {k}: replicas differ"
        assert not torch.equal(a.roll.slab.rewards, b.roll.slab.rewards)
    assert not group.its[0].ppo.exchange.failed()


def test_playback_through_the_inference_policy_and_the_play_script(tmp_path):
    sys.path.insert(0, str(Path(__file__).resolve().parent.parent / "tools"))
    import play_policy
    from wheeledlab_b200.runs import agent_cfg, save_run_config
    env = _env(128)
    r = _runner(env, log_dir=str(tmp_path))
    r.learn(2)
    pol = r.get_inference_policy()
    obs, _ = env.get_observations()
    assert obs.shape == (128, 11)
    from wheeledlab_b200.policy import actor_mean
    assert torch.equal(pol(obs), actor_mean(r.blob, 11, obs, "elu"))
    act = pol(obs)
    o2, *_ = env.step(act)
    assert o2["policy"].shape == (128, 11)
    save_run_config(str(tmp_path), "Isaac-MushrDriftRL-v0", 128, 4, agent_cfg("elu", steps=T, save_interval=1),
                    policy_terms=[(name, fn, nz, cl, None) for name, (fn, nz, cl, _) in zip((t[0] for t in NO_POS_ENV), NO_POS)])
    assert play_policy.main(["-p", str(tmp_path), "--steps", "16"]) == 0
    res = play_policy.resolve(play_policy.parser().parse_args(["-p", str(tmp_path), "--steps", "16"]))
    runner, roll, _ = play_policy.play(res, 16)
    assert roll.table and roll.slab.obs.shape[-1] == 11 and np.array_equal(_bits(runner.blob), _bits(r.blob))
