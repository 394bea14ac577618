"""Host-side event terms on the device (DESIGN 6o): stage b cut in two, the interval timers, the env's event semantics and
training an env that has events.

- wl_step_stage_b1 + wl_step_stage_b2 equal wl_step_stage_b and the fused wl_step bit for bit (obs, reward, dones, state) on
  Drift, F1Tenth, Elevation and Visual over 300 steps with auto-resets and pushes.
- wl_event_timers' fired bytes equal the CPU twin's at N = 1, 33, 4096, 8192 with 1 and 8 terms (lo == hi, hi < step_dt,
  every env reset every step); two shards equal one handle.
- A reset event receives exactly the envs each step reset and its pose write is in that step's observation; env.reset(ids)
  calls it with ids; a startup event runs once; an interval event fires at the ids the twin's timers give.
- No-op events in every mode change nothing over 500 steps; the runner with no-op events equals the fused runner bit for
  bit; with a real interval push it trains with finite losses and resumes from a checkpoint bit for bit."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")


def _sim(task, n, offset=0):
    import wheeledlab_b200 as wl
    sim = wl.WheeledSim(wl.make_task(task, num_envs=n, seed=11, env_id_offset=offset), DEV)
    sim.startup()
    sim.reset(None, 0)
    return sim


def _same(a, b, what):
    assert torch.equal(a.contiguous().view(torch.uint8), b.contiguous().view(torch.uint8)), what


def _step_dt(cfg) -> np.float32:
    import wheeledlab_b200 as wl
    c = type(cfg).from_buffer_copy(cfg)
    assert wl.lib.wl_config_finalize(C.byref(c)) == 0
    return np.float32(c.d_step_dt)


# ---- 1. b1 + b2 == b == the fused step --------------------------------------------------------------------------------
@pytest.mark.parametrize("task,n", [("drift", 256), ("f1tenth_drift", 256), ("elevation", 128), ("visual", 64)])
def test_b1_b2_equal_stage_b_and_the_fused_step(task, n):
    _need_gpu()
    fused, staged, cut = _sim(task, n), _sim(task, n), _sim(task, n)
    g = torch.Generator(device=DEV).manual_seed(3)
    ep = torch.randint(0, int(fused.cfg.max_episode_length), (n,), generator=g, device=DEV, dtype=torch.int32)
    for s in (fused, staged, cut):
        s.episode_length_buf.copy_(ep)                  # time-outs all along the run
    resets = 0
    for t in range(300):
        act = torch.rand((n, 2), generator=g, device=DEV) * 2 - 1
        o0, r0, d0, u0 = fused.step(act, t)
        r1, bits1 = staged.step_stage_a(act, t)
        o1, d1, u1 = staged.step_stage_b(bits1, t)
        r2, bits2 = cut.step_stage_a(act, t)
        d2, u2 = cut.step_stage_b1(bits2, t)
        o2 = cut.step_stage_b2(t)
        for name, x, y, z in (("obs", o0, o1, o2), ("reward", r0, r1, r2), ("terminated", d0, d1, d2), ("truncated", u0, u1, u2)):
            _same(x, y, f"step {t}: {name} (stage b)")
            _same(x, z, f"step {t}: {name} (b1 + b2)")
        resets += int((d0 | u0).sum())
        if t % 50 == 49:
            _same(fused.groups, cut.groups, f"step {t}: state")
            _same(staged.groups, cut.groups, f"step {t}: state (stage b)")
    assert resets > n // 2, "the run must auto-reset"


def test_b2_refuses_a_counter_b1_was_not_given():
    _need_gpu()
    from wheeledlab_b200._lib import WlError
    sim = _sim("drift", 64)
    act = torch.zeros((64, 2), device=DEV)
    _, bits = sim.step_stage_a(act, 0)
    sim.step_stage_b1(bits, 0)
    with pytest.raises(WlError, match="wl_step_stage_b2"):
        sim.step_stage_b2(1)
    sim.step_stage_b2(0)


# ---- 2. the interval timers against the twin ------------------------------------------------------------------------
RANGES8 = [(0.5, 1.0), (0.0, 0.0), (0.1, 0.1), (0.02, 0.05), (2.0, 3.0), (0.3, 0.9), (0.0, 0.05), (1.0, 1.5)]


@pytest.mark.parametrize("n", [1, 33, 4096, 8192])
@pytest.mark.parametrize("ranges", [RANGES8[:1], RANGES8[1:2], RANGES8], ids=["1 term", "1 term lo == hi == 0", "8 terms"])
def test_event_timers_equal_the_twin(n, ranges):
    _need_gpu()
    import event_timers_oracle as eo
    sim = _sim("drift", n)
    seed, dt = int(sim.cfg.seed), _step_dt(sim.cfg)
    sim.set_event_timers(ranges)
    tl = eo.init(seed, 0, n, ranges)
    fired = torch.empty((len(ranges), n), dtype=torch.uint8, device=DEV)
    rng = np.random.default_rng(n)
    fires = 0
    for t in range(120):
        done = np.ones(n, np.uint8) if 5 <= t < 15 else (rng.random(n) < 0.02).astype(np.uint8)   # (5..14: every env every step)
        sim.event_timers(torch.from_numpy(done).to(DEV), t, fired)
        want = eo.step(seed, 0, ranges, dt, done, tl, t)
        assert np.array_equal(fired.cpu().numpy(), want), t
        fires += int(want.sum())
    assert fires > 0 or n == 1


def test_event_timers_do_not_depend_on_sharding():
    _need_gpu()
    n, ranges = 4096, RANGES8
    whole, halves = _sim("drift", n), [_sim("drift", n // 2, 0), _sim("drift", n // 2, n // 2)]
    for s in [whole] + halves:
        s.set_event_timers(ranges)
    f = torch.empty((8, n), dtype=torch.uint8, device=DEV)
    fh = [torch.empty((8, n // 2), dtype=torch.uint8, device=DEV) for _ in halves]
    g = torch.Generator(device=DEV).manual_seed(1)
    for t in range(40):
        done = (torch.rand(n, generator=g, device=DEV) < 0.1).to(torch.uint8)
        whole.event_timers(done, t, f)
        for h, s in enumerate(halves):
            s.event_timers(done[h * n // 2:(h + 1) * n // 2].contiguous(), t, fh[h])
        _same(f, torch.cat(fh, dim=1), f"step {t}")


def test_event_timer_refusals():
    _need_gpu()
    from wheeledlab_b200._lib import WlError
    sim = _sim("drift", 64)
    f = torch.empty((1, 64), dtype=torch.uint8, device=DEV)
    with pytest.raises(WlError, match="no event timers"):
        sim.event_timers(torch.zeros(64, dtype=torch.uint8, device=DEV), 0, f)
    for bad in ([(1.0, 0.5)], [(-0.1, 1.0)], [(0.0, float("nan"))], [(0.1, 0.2)] * 9):
        with pytest.raises(WlError, match="wl_set_event_timers"):
            sim.set_event_timers(bad)
    sim.set_event_timers([(0.1, 0.2)])
    sim.set_event_timers([])
    with pytest.raises(WlError, match="no event timers"):
        sim.event_timers(torch.zeros(64, dtype=torch.uint8, device=DEV), 0, f)


# ---- 3. the env's event semantics ------------------------------------------------------------------------------------
def _env(n=256, task="Isaac-MushrDriftRL-v0", **kw):
    import wheeledlab_b200 as wl
    return wl.make(task, device=DEV, num_envs=n, seed=5, **kw)


def test_reset_startup_and_interval_event_semantics():
    _need_gpu()
    import event_timers_oracle as eo
    n = 256
    env = _env(n)
    log = {"startup": [], "reset": [], "kick": []}

    def on_start(e, ids):
        log["startup"].append(ids)

    def on_reset(e, ids, x=50.0):             # even envs to x (off the track: they reset again next step), odd ones kept
        log["reset"].append(ids.clone())
        sel = ids[ids % 2 == 0]
        pose = torch.zeros((sel.numel(), 7), device=DEV)
        pose[:, 0], pose[:, 3] = x, 1.0
        e.scene["robot"].write_root_pose_to_sim(pose, env_ids=sel)

    def on_kick(e, ids):
        log["kick"].append(ids.clone())

    env.add_event_term("boot", on_start, "startup")
    assert log["startup"] == [None]
    env.add_event_term("spawn", on_reset, "reset", {"x": 50.0})
    ranges = [(0.1, 0.5)]
    env.add_event_term("kick", on_kick, "interval", interval_range_s=ranges[0])
    tl = eo.init(int(env.spec.cfg.seed), 0, n, ranges)
    dt = _step_dt(env.spec.cfg)
    env.reset()
    _same(log["reset"].pop(), torch.arange(n, device=DEV), "reset() calls the reset events with every env")
    env.episode_length_buf = torch.randint(0, int(env.max_episode_length), (n,), device=DEV)
    g = torch.Generator(device=DEV).manual_seed(2)
    resets = kicks = 0
    for t in range(120):
        obs, rew, term, trunc, _ = env.step(torch.rand((n, 2), generator=g, device=DEV) * 2 - 1)
        done = (term | trunc)
        ids = done.nonzero().squeeze(1)
        if ids.numel():
            got = log["reset"].pop()
            _same(got, ids, f"step {t}: reset ids")
            assert got.dtype == torch.int64
            p, even = obs["policy"], ids[ids % 2 == 0]
            if even.numel():
                assert (p[even, 0] - 50.0).abs().max() < 1.0, "the event's pose write is in this step's observation"
            assert (p[ids[ids % 2 == 1], 0]).abs().le(20.0).all()
            resets += ids.numel()
        assert not log["reset"], f"step {t}: the reset event ran without resets"
        fired = eo.step(int(env.spec.cfg.seed), 0, ranges, dt, done.to(torch.uint8).cpu().numpy(), tl, t)
        want = torch.from_numpy(np.nonzero(fired[0])[0]).to(DEV)
        if want.numel():
            _same(log["kick"].pop(), want, f"step {t}: interval ids")
            kicks += 1
        assert not log["kick"], f"step {t}: the interval event ran without firing"
    assert resets > 0 and kicks > 0
    assert log["startup"] == [None], "the startup event runs once"
    some = torch.tensor([7, 3, 100], device=DEV)
    obs, _ = env.reset(env_ids=some)
    _same(log["reset"].pop(), some, "reset(ids) calls the reset events with ids")
    assert (obs["policy"][100, 0] - 50.0).abs() < 1.0 and obs["policy"][[7, 3], 0].abs().le(20.0).all()


@pytest.mark.parametrize("task,n", [("Isaac-MushrDriftRL-v0", 256), ("Isaac-MushrElevationRL-v0", 64)])
def test_noop_events_change_nothing(task, n):
    _need_gpu()
    plain, ev = _env(n, task), _env(n, task)
    calls = []
    ev.add_event_term("s", lambda e, ids: calls.append("s"), "startup")
    ev.add_event_term("r", lambda e, ids: calls.append("r"), "reset")
    ev.add_event_term("i", lambda e, ids: calls.append("i"), "interval", interval_range_s=(0.0, 0.3))
    for e in (plain, ev):
        e.reset()
        e.episode_length_buf = torch.arange(n, device=DEV) % int(e.max_episode_length)
    g = torch.Generator(device=DEV).manual_seed(4)
    for t in range(500):
        act = torch.rand((n, 2), generator=g, device=DEV) * 2 - 1
        a, b = plain.step(act), ev.step(act)
        for name, x, y in (("obs", a[0]["policy"], b[0]["policy"]), ("reward", a[1], b[1]), ("terminated", a[2], b[2]),
                           ("truncated", a[3], b[3])):
            _same(x, y, f"step {t}: {name}")
    _same(plain.sim.groups, ev.sim.groups, "state")
    assert {"s", "r", "i"} <= set(calls)


# ---- 4. training ---------------------------------------------------------------------------------------------------
T = 16


def _runner(env, seed, **kw):
    from wheeledlab_b200.learner import FusedOnPolicyRunner
    from wheeledlab_b200.runs import agent_cfg
    torch.manual_seed(seed)
    return FusedOnPolicyRunner(env, agent_cfg("elu", steps=T, save_interval=1), device=DEV, **kw)


def _noop_events(env):
    env.add_event_term("s", lambda e, ids: None, "startup")
    env.add_event_term("r", lambda e, ids: None, "reset")
    env.add_event_term("i", lambda e, ids: None, "interval", interval_range_s=(0.0, 0.3))
    return env


def _kick(env, ids, speed=0.5):
    robot = env.scene["robot"]
    vel = torch.cat([robot.data.root_lin_vel_w[ids], robot.data.root_ang_vel_w[ids]], dim=1)
    vel[:, 0] += speed
    robot.write_root_velocity_to_sim(vel, env_ids=ids)


def _kick_env(n=256):
    env = _env(n)
    env.add_event_term("kick", _kick, "interval", {"speed": 0.5}, interval_range_s=(0.2, 0.6))
    return env


def test_noop_events_train_like_the_fused_runner():
    _need_gpu()
    from wheeledlab_b200.learner import StagedPPOIteration
    fused_env, ev_env = _env(), _noop_events(_env())
    fused, staged = _runner(fused_env, 3), _runner(ev_env, 3)
    assert isinstance(staged.it, StagedPPOIteration) and not isinstance(fused.it, StagedPPOIteration)
    logs = []
    for r in (fused, staged):
        torch.manual_seed(17)
        logs.append(r.learn(3))
    torch.cuda.synchronize()
    assert fused_env.common_step_counter == ev_env.common_step_counter == 3 * T
    for name, x, y in (("slab", fused.it.roll.slab.flat, staged.it.roll.slab.flat), ("blob", fused.blob, staged.blob),
                       ("adam m", fused.alg.m, staged.alg.m), ("adam v", fused.alg.v, staged.alg.v),
                       ("ppo state", fused.alg.state, staged.alg.state), ("env state", fused_env.sim.groups, ev_env.sim.groups),
                       ("episode statistics", fused.it.episodes.state, staged.it.episodes.state),
                       ("episode-log rows", fused.it.roll.logs, staged.it.roll.logs)):
        _same(x, y, name)
    a, b = logs
    assert set(a) == set(b)
    for k in a:
        if k != "Perf/total_fps":
            assert a[k] == b[k], k


def test_interval_push_trains_and_resumes(tmp_path):
    _need_gpu()
    from wheeledlab_b200.learner import FusedOnPolicyRunner
    from wheeledlab_b200.runs import agent_cfg
    env_a, env_b = _kick_env(), _kick_env()
    a, b = _runner(env_a, 6, log_dir=str(tmp_path)), _runner(env_b, 6)
    blob0 = a.blob.clone()
    for r in (a, b):
        torch.manual_seed(21)
        log = r.learn(2)
        assert all(math.isfinite(v) for k, v in log.items() if k.startswith("Loss/")), log
    assert not torch.equal(blob0, a.blob)
    c = FusedOnPolicyRunner(env_b, agent_cfg("elu", steps=T, save_interval=1), device=DEV)
    c.load(str(tmp_path / "models" / "model_1.pt"))
    a.alg.state[0] = c.alg.cfg.learning_rate               # (a load restarts the adaptive rate from the cfg's)
    for r in (a, c):
        torch.manual_seed(22)
        r.learn(1)
    torch.cuda.synchronize()
    assert env_a.common_step_counter == env_b.common_step_counter == 3 * T
    for name, x, y in (("blob", a.blob, c.blob), ("m", a.alg.m, c.alg.m), ("v", a.alg.v, c.alg.v)):
        _same(x, y, name)


def test_events_keep_the_runner_and_env_refusals():
    _need_gpu()
    env = _noop_events(_env(64))
    with pytest.raises(NotImplementedError, match="step_host"):
        env.step_host(torch.zeros((64, 2)))
    with pytest.raises(NotImplementedError, match="a critic observation group together with host-side Python terms"):
        env.set_critic_observation(["root_pos_w"])
    with pytest.raises(NotImplementedError, match="either device terms or host-side Python"):
        from wheeledlab_b200.device_terms import REGISTRY
        env.add_device_reward_term("x", next(iter(REGISTRY)), 1.0)
    with pytest.raises(NotImplementedError, match="event term bad: mode 'prestartup'"):
        env.add_event_term("bad", lambda e, ids: None, "prestartup")
    for k in range(7):
        env.add_event_term(f"i{k}", lambda e, ids: None, "interval", interval_range_s=(0.1, 0.2))
    with pytest.raises(NotImplementedError, match="more than 8 Python interval event terms"):
        env.add_event_term("i8", lambda e, ids: None, "interval", interval_range_s=(0.1, 0.2))
