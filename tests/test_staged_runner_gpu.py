"""Training an env that has host-side Python reward / termination terms: wl_policy_act_elu against wl_act_step, the staged
rollout against the eager loop of policy_act + env.step, and FusedOnPolicyRunner on it.

- wl_policy_act_elu stores what wl_act_step stores (actions, mean, log-prob, value) bit for bit, on Drift, F1Tenth and the
  8-float Visual spec, at N = 1, 31, 33, 4096 and 33 793 (partial CTAs either side of 32), under a host counter, a device
  counter replayed in a CUDA graph and a nonzero env_id_offset; bad arguments and a set fan-out are refused before any
  launch.
- No-op Python terms (a reward of weight 0, a termination that never fires) change nothing: the staged runner's slab,
  blob, Adam moments and state, env state, episode statistics and built-in log entries equal the fused runner's, bit for
  bit, on Drift (ELU) and Elevation (ReLU).
- Real terms: the runner's slab equals the eager loop's, its Episode_Reward/<name> and Episode_Termination/<name> are the
  T-step means of the loop's extras["log"], and a checkpoint resumes to the same blob as an uninterrupted run."""
import ctypes as C

import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")


def _blob(obs_dim, seed=0):
    from wheeledlab_b200.policy import pack_actor_critic
    torch.manual_seed(seed)
    mk = lambda out: torch.nn.Sequential(torch.nn.Linear(obs_dim, 64), torch.nn.ELU(), torch.nn.Linear(64, 64), torch.nn.ELU(),
                                         torch.nn.Linear(64, out))
    return pack_actor_critic(mk(2), mk(1), torch.tensor([0.7, 1.3]), obs_dim, DEV)


def _sim(task, n, offset=0):
    import wheeledlab_b200 as wl
    sim = wl.WheeledSim(wl.make_task(task, num_envs=n, seed=11, env_id_offset=offset), DEV)
    sim.startup()
    sim.reset(None, 0)
    return sim


def _outs(n):
    return [torch.full((n, 2), float("nan"), device=DEV), torch.full((n, 2), float("nan"), device=DEV),
            torch.full((n,), float("nan"), device=DEV), torch.full((n,), float("nan"), device=DEV)]


def _same(a, b, what):
    assert torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32)), what


# ---- 1. the kernel contract -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("task,n,offset", [("drift", 1, 0), ("drift", 31, 0), ("drift", 33, 0), ("drift", 4096, 0), ("drift", 33793, 0),
                                           ("f1tenth_drift", 33, 0), ("f1tenth_drift", 4096, 0), ("visual", 31, 0), ("visual", 4096, 0),
                                           ("drift", 4096, 70001), ("visual", 33, 123)])
def test_policy_act_elu_equals_act_step(task, n, offset):
    """Each step: wl_policy_act_elu on the act step's obs_in and counter, then wl_act_step; the four outputs bit for bit."""
    _need_gpu()
    from wheeledlab_b200.policy import act_step, policy_act
    sim = _sim(task, n, offset)
    D = sim.obs_dim
    assert D <= 16
    blob = _blob(D)
    obs_in = sim.observe(0, 0)
    out = (torch.empty((n, D), device=DEV), torch.empty(n, device=DEV), torch.empty(n, dtype=torch.uint8, device=DEV),
           torch.empty(n, dtype=torch.uint8, device=DEV))
    for t in range(4):
        mine, fused = _outs(n), _outs(n)
        policy_act(sim, obs_in, blob, *mine, t, activation="elu")
        act_step(sim, obs_in, blob, *fused, out, None, t)
        for name, x, y in zip(("actions", "mean", "log_prob", "value"), mine, fused):
            _same(x, y, f"{task} N={n} offset={offset} step {t}: {name}")
        obs_in = out[0].clone()


def test_policy_act_elu_device_counter_in_a_graph():
    """WL_DEVICE_COUNTER_PLUS(k) replayed in a CUDA graph equals the host counter base + k, across two replays."""
    _need_gpu()
    from wheeledlab_b200 import WheeledSim
    from wheeledlab_b200.policy import policy_act
    n, K = 4096, 3
    sim = _sim("drift", n)
    blob = _blob(sim.obs_dim, seed=1)
    g = torch.Generator(device=DEV).manual_seed(5)
    obs = [torch.randn((n, sim.obs_dim), device=DEV, generator=g) for _ in range(K)]
    outs = [_outs(n) for _ in range(K)]
    base = 1000
    sim.set_step_counter(base)
    graph, s = torch.cuda.CUDAGraph(), torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s), torch.cuda.graph(graph, stream=s):
        for k in range(K):
            policy_act(sim, obs[k], blob, *outs[k], WheeledSim.device_counter_plus(k), activation="elu")
        sim.advance_counter(K)
    torch.cuda.current_stream().wait_stream(s)
    sim.set_step_counter(base)
    for rep in range(2):
        graph.replay()
        for k in range(K):
            ref = _outs(n)
            policy_act(sim, obs[k], blob, *ref, base + rep * K + k, activation="elu")
            for name, x, y in zip(("actions", "mean", "log_prob", "value"), outs[k], ref):
                _same(x, y, f"replay {rep} k {k}: {name}")


def test_policy_act_elu_refusals_launch_nothing():
    _need_gpu()
    import wheeledlab_b200 as wl
    from wheeledlab_b200._lib import WlPolicyOut, lib
    n = 64
    sim = _sim("drift", n)
    blob = _blob(sim.obs_dim)
    obs = sim.observe(0, 0)
    a, m, lp, v = _outs(n)
    p = lambda x, off=0: C.c_void_p(x.data_ptr() + off)
    good = WlPolicyOut(a.data_ptr(), m.data_ptr(), lp.data_ptr(), v.data_ptr())
    cases = [
        ("null handle", (None, p(obs), p(blob), good, 0), -1),
        ("null obs_in", (sim._h, None, p(blob), good, 0), -1),
        ("null blob", (sim._h, p(obs), None, good, 0), -1),
        ("null actions", (sim._h, p(obs), p(blob), WlPolicyOut(0, m.data_ptr(), lp.data_ptr(), v.data_ptr()), 0), -1),
        ("null value", (sim._h, p(obs), p(blob), WlPolicyOut(a.data_ptr(), m.data_ptr(), lp.data_ptr(), 0), 0), -1),
        ("blob not 16-aligned", (sim._h, p(obs), p(blob, 4), good, 0), -1),
        ("actions not 8-aligned", (sim._h, p(obs), p(blob), WlPolicyOut(a.data_ptr() + 4, m.data_ptr(), lp.data_ptr(), v.data_ptr()), 0), -1),
        ("mean not 8-aligned", (sim._h, p(obs), p(blob), WlPolicyOut(a.data_ptr(), m.data_ptr() + 4, lp.data_ptr(), v.data_ptr()), 0), -1),
        ("obs_in not 4-aligned", (sim._h, p(obs, 2), p(blob), good, 0), -1),
        ("log_prob not 4-aligned", (sim._h, p(obs), p(blob), WlPolicyOut(a.data_ptr(), m.data_ptr(), lp.data_ptr() + 1, v.data_ptr()), 0), -1),
        ("counter >= 2^31", (sim._h, p(obs), p(blob), good, 1 << 31), -1),
    ]
    before = sim.launch_count
    for what, args, rc in cases:
        assert lib.wl_policy_act_elu(*args, None) == rc, what
        assert b"wl_policy_act_elu" in lib.wl_last_error(), what
    # a peer fan-out, then the multicast one on top: refused (the staged step that follows refuses them too)
    sim.set_peer_fanout([1 << 20])
    assert lib.wl_policy_act_elu(sim._h, p(obs), p(blob), good, 0, None) == -3
    assert b"fan-out" in lib.wl_last_error()
    sim.set_multicast_fanout(1 << 21)
    assert lib.wl_policy_act_elu(sim._h, p(obs), p(blob), good, 0, None) == -3
    sim.set_peer_fanout([])
    assert sim.launch_count == before, "a refused call launched"
    torch.cuda.synchronize()
    assert torch.isnan(a).all() and torch.isnan(v).all(), "a refused call wrote outputs"
    # obs_dim > 16 (Elevation's 689 floats): the ELU network is wl_act_step's
    elev = wl.WheeledSim(wl.make_task("elevation", num_envs=32, seed=3), DEV)
    eb = torch.zeros(lib.wl_policy_blob_floats(elev.obs_dim, None), device=DEV)
    eo = torch.zeros((32, elev.obs_dim), device=DEV)
    n0 = elev.launch_count
    assert lib.wl_policy_act_elu(elev._h, p(eo), p(eb), good, 0, None) == -3
    assert b"obs_dim" in lib.wl_last_error() and elev.launch_count == n0
    # the accepted call launches once
    lib.wl_policy_act_elu(sim._h, p(obs), p(blob), good, 0, None)
    assert sim.launch_count == before + 1
    torch.cuda.synchronize()
    assert not torch.isnan(a).any()


# ---- 2.-4. the runner on the staged rollout ----------------------------------------------------------------------------
T = 16


def _forward_speed(env):
    return env.scene["robot"].data.root_lin_vel_b[:, 0]


def _never(env):
    return torch.zeros(env.num_envs, dtype=torch.bool, device=env.device)


def _long_episode(env):
    return env.episode_length_buf >= 7


def _env(task, n, terms):
    import wheeledlab_b200 as wl
    env = wl.make(task, device=DEV, num_envs=n, seed=5)
    if terms == "noop":
        env.add_reward_term("zero_weight", _forward_speed, 0.0)
        env.add_termination_term("never", _never)
    elif terms == "real":
        env.add_reward_term("forward_speed", _forward_speed, 0.5)
        env.add_termination_term("long_episode", _long_episode)
    return env


def _runner(env, activation, seed, **kw):
    from wheeledlab_b200.learner import FusedOnPolicyRunner
    from wheeledlab_b200.runs import agent_cfg
    torch.manual_seed(seed)
    return FusedOnPolicyRunner(env, agent_cfg(activation, steps=T, save_interval=1), device=DEV, **kw)


@pytest.mark.parametrize("task,n,activation", [("Isaac-MushrDriftRL-v0", 256, "elu"), ("Isaac-MushrElevationRL-v0", 64, "relu")])
def test_noop_python_terms_train_like_the_fused_runner(task, n, activation):
    _need_gpu()
    from wheeledlab_b200.learner import StagedPPOIteration
    fused_env, staged_env = _env(task, n, None), _env(task, n, "noop")
    fused, staged = _runner(fused_env, activation, 3), _runner(staged_env, activation, 3)
    assert isinstance(staged.it, StagedPPOIteration) and not isinstance(fused.it, StagedPPOIteration)
    logs = []
    for r in (fused, staged):
        torch.manual_seed(17)
        logs.append(r.learn(2))
    torch.cuda.synchronize()
    assert fused_env.common_step_counter == staged_env.common_step_counter == 2 * T
    for name, x, y in (("slab", fused.it.roll.slab.flat, staged.it.roll.slab.flat), ("blob", fused.blob, staged.blob),
                       ("adam m", fused.alg.m, staged.alg.m), ("adam v", fused.alg.v, staged.alg.v),
                       ("ppo state", fused.alg.state, staged.alg.state), ("env state", fused_env.sim.groups, staged_env.sim.groups),
                       ("reward weights", fused_env.sim.rew_weight, staged_env.sim.rew_weight),
                       ("episode statistics", fused.it.episodes.state, staged.it.episodes.state),
                       ("running returns", fused.it.episodes.cur_return, staged.it.episodes.cur_return),
                       ("running lengths", fused.it.episodes.cur_length, staged.it.episodes.cur_length),
                       ("episode-log rows", fused.it.roll.logs, staged.it.roll.logs)):
        assert torch.equal(x.view(torch.uint8), y.view(torch.uint8)), name
    a, b = logs
    assert set(b) == set(a) | {"Episode_Reward/zero_weight", "Episode_Termination/never"}
    assert b["Episode_Reward/zero_weight"] == 0.0 and b["Episode_Termination/never"] == 0.0
    for k in a:
        if k != "Perf/total_fps":
            assert a[k] == b[k], k


def test_python_terms_rollout_equals_the_eager_loop():
    """Iteration 0 of the runner against a hand-written loop of policy_act + env.step over an identical env."""
    _need_gpu()
    from wheeledlab_b200.policy import policy_act
    n = 256
    env = _env("Isaac-MushrDriftRL-v0", n, "real")
    runner = _runner(env, "elu", 4)
    blob0 = runner.blob.clone()
    torch.manual_seed(8)
    log = runner.learn(1)
    torch.cuda.synchronize()
    slab = runner.it.roll.slab
    # the loop
    loop_env = _env("Isaac-MushrDriftRL-v0", n, "real")
    loop_env.reset()
    D = loop_env.sim.obs_dim
    obs = loop_env.sim.observe(loop_env.common_step_counter, 0)
    names = ["Episode_Reward/forward_speed", "Episode_Termination/long_episode"]
    fired, rows = 0, []
    for k in range(T):
        act, mean = torch.empty((n, 2), device=DEV), torch.empty((n, 2), device=DEV)
        lp, val = torch.empty(n, device=DEV), torch.empty(n, device=DEV)
        _same(obs, slab.obs_in[k], f"step {k}: obs_in")
        policy_act(loop_env.sim, obs, blob0, act, mean, lp, val, loop_env.common_step_counter, activation="elu")
        o, rew, term, trunc, extras = loop_env.step(act)
        for name, x, y in (("actions", act, slab.actions[k]), ("mean", mean, slab.mean[k]), ("log_prob", lp, slab.log_prob[k]),
                           ("values", val, slab.values[k]), ("rewards", rew, slab.rewards[k]), ("obs", o["policy"], slab.obs[k])):
            _same(x, y, f"step {k}: {name}")
        assert torch.equal(term.view(torch.uint8), slab.terminated[k]) and torch.equal(trunc.view(torch.uint8), slab.truncated[k]), k
        fired += int(loop_env.termination_manager.get_term("long_episode").sum())
        rows.append(torch.stack([extras["log"][name].to(torch.float64) for name in names]))
        obs = o["policy"].clone()
    assert fired > 0, "the termination term must fire mid-rollout"
    assert loop_env.common_step_counter == env.common_step_counter == T
    means = torch.stack(rows).cpu().mean(0).tolist()
    for name, want in zip(names, means):
        assert log[name] == want, name
    assert log["Episode_Termination/long_episode"] > 0
    assert not torch.equal(blob0, runner.blob), "the update did not move the weights"


def test_python_terms_checkpoint_resumes_bit_for_bit(tmp_path):
    _need_gpu()
    from wheeledlab_b200.learner import FusedOnPolicyRunner
    from wheeledlab_b200.runs import agent_cfg
    env_a, env_b = _env("Isaac-MushrDriftRL-v0", 256, "real"), _env("Isaac-MushrDriftRL-v0", 256, "real")
    a, b = _runner(env_a, "elu", 6, log_dir=str(tmp_path)), _runner(env_b, "elu", 6)
    for r in (a, b):
        torch.manual_seed(21)
        r.learn(2)                                          # a writes models/model_0.pt and model_1.pt
    c = FusedOnPolicyRunner(env_b, agent_cfg("elu", steps=T, save_interval=1), device=DEV)
    c.load(str(tmp_path / "models" / "model_1.pt"))
    assert c.current_learning_iteration == 1
    a.alg.state[0] = c.alg.cfg.learning_rate               # (a load restarts the adaptive rate from the cfg's)
    for r in (a, c):
        torch.manual_seed(22)
        r.learn(1)
    torch.cuda.synchronize()
    assert env_a.common_step_counter == env_b.common_step_counter == 3 * T
    for name, x, y in (("blob", a.blob, c.blob), ("m", a.alg.m, c.alg.m), ("v", a.alg.v, c.alg.v)):
        _same(x, y, name)


def test_runner_refuses_python_observation_terms():
    _need_gpu()
    env = _env("Isaac-MushrDriftRL-v0", 64, "real")
    env.add_observation_term("speed", lambda e: _forward_speed(e).unsqueeze(1))
    with pytest.raises(NotImplementedError, match="Python observation terms"):
        _runner(env, "elu", 0)
