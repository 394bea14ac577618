"""Device event terms (wl_set_device_events / wl_device_events / wl_step_terms, DESIGN 6p) on the GPU:

- wl_device_events equals the oracle's twin (wlo_device_events) bit for bit on every task at N = 1, 33, 4096, 8192
  with 1 and 8 terms (an interval range of (0, 0), which fires every step; every env reset every tenth step), and two
  shards equal one handle;
- the whole step with device events equals the step without them plus the twin's push on its state, step after step, on
  every task and together with device terms;
- all-zero ranges leave the env as it is without events, bit for bit over 500 steps (Drift, Elevation);
- a captured graph of device-counter steps equals the same steps run eagerly;
- the runner trains an Elevation env with an interval push in one graph, and a checkpoint resumes it bit for bit;
- the calls that would step the handle without its events refuse it."""
import ctypes as C
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
from wheeledlab_b200.env import ManagerBasedRLEnv              # noqa: E402
from wheeledlab_b200.sim import G_ANGVEL, G_LINVEL, WheeledSim  # noqa: E402

DEV = "cuda:0"
TASKS = ["drift", "f1tenth_drift", "elevation", "visual"]
PUSH = [(-0.5, 0.5), (-0.25, 0.25), (0.0, 0.1), (-0.2, 0.2), (-0.2, 0.2), (-1.0, 1.0)]
ZERO = [(0.0, 0.0)] * 6
TABLE_1 = [("interval", (0.0, 0.15), PUSH)]          # (fires within the Drift family's reset period too)
TABLE_8 = [("interval", (0.2, 0.6), PUSH), ("reset", None, [(-1.0, 1.0)] * 6), ("interval", (0.0, 0.0), [(0.01, 0.02)] * 6),
           ("interval", (0.05, 0.3), [(0.1, 0.2), (-0.3, -0.1), (0.0, 0.0), (0.5, 0.5), (-2.0, 2.0), (0.0, 1.0)]),
           ("reset", None, ZERO), ("interval", (1.0, 2.0), PUSH), ("interval", (0.0, 0.05), [(-0.01, 0.0)] * 6),
           ("reset", None, [(0.0, 0.3)] * 6)]


def _push():
    root = Path(__file__).resolve().parent.parent
    if str(root / "shims") not in sys.path:
        sys.path.insert(0, str(root / "shims"))
    from isaaclab.envs import mdp
    return mdp.push_by_setting_velocity


def _vr(ranges):
    return {"velocity_range": {c: r for c, r in zip(("x", "y", "z", "roll", "pitch", "yaw"), ranges)}}


def _sim(task, n, offset=0, table=None):
    sim = WheeledSim(wl.make_task(task, num_envs=n, seed=11, env_id_offset=offset), DEV)
    if table:
        sim.set_device_events(table)
    sim.startup()
    sim.reset(None, 0)
    return sim


def _step_dt(cfg) -> np.float32:
    c = type(cfg).from_buffer_copy(cfg)
    assert wl.lib.wl_config_finalize(C.byref(c)) == 0
    return np.float32(c.d_step_dt)


def _vel(sim) -> np.ndarray:
    return torch.cat([sim.groups[G_LINVEL, :, 0:3], sim.groups[G_ANGVEL, :, 0:3]], dim=1).cpu().numpy().copy()


def _bits(x):
    return x.contiguous().view(torch.uint8)


def _done(rng, n, t):
    """(terminated, truncated) u8: every env on every tenth step, else about one in ten."""
    if t % 10 == 9:
        return np.ones(n, np.uint8), (rng.random(n) < 0.5).astype(np.uint8)
    return (rng.random(n) < 0.05).astype(np.uint8), (rng.random(n) < 0.05).astype(np.uint8)


# ---- 1. the kernel against the twin ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("task", TASKS)
@pytest.mark.parametrize("n", [1, 33, 4096, 8192])
@pytest.mark.parametrize("table", [TABLE_1, TABLE_8], ids=["1term", "8terms"])
def test_kernel_equals_the_twin(task, n, table):
    from oracle_lib import device_events_init, device_events_step
    sim = _sim(task, n, table=table)
    gen = torch.Generator(device=DEV).manual_seed(n)
    sim.groups[G_LINVEL, :, 0:3] = torch.randn((n, 3), device=DEV, generator=gen)
    sim.groups[G_ANGVEL, :, 0:3] = torch.randn((n, 3), device=DEV, generator=gen)
    w_before = torch.stack([sim.groups[G_LINVEL, :, 3], sim.groups[G_ANGVEL, :, 3]]).clone()
    seed, dt = int(sim.cfg.seed), _step_dt(sim.cfg)
    tl, vel = device_events_init(seed, 0, n, table), _vel(sim)
    rng = np.random.default_rng(7)
    moved = 0
    for t in range(40):
        term, trunc = _done(rng, n, t)
        sim.device_events(torch.from_numpy(term).to(DEV), torch.from_numpy(trunc).to(DEV), t)
        before = vel.copy()
        device_events_step(seed, 0, table, dt, term | trunc, tl, vel, t)
        got = _vel(sim)
        assert np.array_equal(got.view(np.uint32), vel.view(np.uint32)), f"step {t}"
        moved += int((before != vel).any(axis=1).sum())
    assert moved > 0
    w_after = torch.stack([sim.groups[G_LINVEL, :, 3], sim.groups[G_ANGVEL, :, 3]])
    assert torch.equal(w_before, w_after), "the built-in push timers are not the kernel's"


def test_two_shards_equal_one_handle():
    n = 4096
    whole = _sim("elevation", n, table=TABLE_8)
    halves = [_sim("elevation", n // 2, offset=h * (n // 2), table=TABLE_8) for h in (0, 1)]
    gen = torch.Generator(device=DEV).manual_seed(1)
    v0 = torch.randn((2, n, 3), device=DEV, generator=gen)
    whole.groups[G_LINVEL, :, 0:3], whole.groups[G_ANGVEL, :, 0:3] = v0[0], v0[1]
    for h, s in enumerate(halves):
        sl = slice(h * (n // 2), (h + 1) * (n // 2))
        s.groups[G_LINVEL, :, 0:3], s.groups[G_ANGVEL, :, 0:3] = v0[0, sl], v0[1, sl]
    rng = np.random.default_rng(3)
    for t in range(30):
        term, trunc = (torch.from_numpy(x).to(DEV) for x in _done(rng, n, t))
        whole.device_events(term, trunc, t)
        for h, s in enumerate(halves):
            sl = slice(h * (n // 2), (h + 1) * (n // 2))
            s.device_events(term[sl].contiguous(), trunc[sl].contiguous(), t)
    assert np.array_equal(_vel(whole), np.concatenate([_vel(s) for s in halves]))


# ---- 2. the whole step: without the events, plus the twin's push -------------------------------------------------------------
def _add_terms(env):
    from wheeledlab_b200 import device_terms as dtm
    env.add_device_reward_term("steep", dtm.resolve("steep_penalty", dtm.ELEVATION), -1.0, {"thresh_pitch": 0.05})
    env.add_device_termination_term("flip", dtm.resolve("roll_over", dtm.VISUAL))


@pytest.mark.parametrize("task,terms", [("drift", False), ("f1tenth_drift", False), ("elevation", False), ("visual", False),
                                        ("elevation", True), ("drift", True)])
def test_the_step_is_the_step_without_events_plus_the_twins_push(task, terms):
    """Each step: B takes A's state, both step (A with the events), and A's state equals B's with the twin's push applied
    for B's done bytes; rewards and dones are equal (the events come after them).  With device terms on both."""
    from oracle_lib import device_events_init, device_events_step
    n = 256
    spec = lambda: wl.make_task(task, num_envs=n, seed=5)
    a, b = ManagerBasedRLEnv(spec(), device=DEV), ManagerBasedRLEnv(spec(), device=DEV)
    if terms:
        _add_terms(a); _add_terms(b)
    table = [("interval", (0.1, 0.3), PUSH), ("reset", None, [(0.0, 0.5)] * 6), ("interval", (0.0, 0.0), [(-0.01, 0.01)] * 6)]
    for k, (mode, rng_s, ranges) in enumerate(table):
        a.add_device_event_term(f"push{k}", _push(), mode, rng_s, _vr(ranges))
    for e in (a, b):
        e.reset()
    seed, dt = int(a.spec.cfg.seed), _step_dt(a.spec.cfg)
    tl = device_events_init(seed, 0, n, table)
    gen = torch.Generator(device=DEV).manual_seed(2)
    fired = 0
    for t in range(120):
        b.sim.groups.copy_(a.sim.groups)
        act = torch.rand((n, 2), device=DEV, generator=gen) * 2 - 1
        _, ra, ta, ua, _ = a.step(act)
        _, rb, tb, ub, _ = b.step(act)
        torch.cuda.synchronize()
        assert torch.equal(_bits(ra), _bits(rb)) and torch.equal(ta, tb) and torch.equal(ua, ub), f"step {t}"
        vel = _vel(b.sim)
        before = vel.copy()
        device_events_step(seed, 0, table, dt, (tb | ub).cpu().numpy().astype(np.uint8), tl, vel, t)
        assert np.array_equal(_vel(a.sim).view(np.uint32), vel.view(np.uint32)), f"step {t}"
        rest = [g for g in range(a.sim.groups.shape[0]) if g not in (G_LINVEL, G_ANGVEL)]
        assert torch.equal(a.sim.groups[rest], b.sim.groups[rest]), f"step {t}"
        fired += int((before != vel).any(axis=1).sum())
    assert fired > 0 and a.common_step_counter == 120


# ---- 3. all-zero ranges: the env without events ---------------------------------------------------------------------------
@pytest.mark.parametrize("task", ["drift", "elevation"])
def test_all_zero_ranges_equal_the_env_without_events(task):
    n = 256
    a = ManagerBasedRLEnv(wl.make_task(task, num_envs=n, seed=8), device=DEV)
    b = ManagerBasedRLEnv(wl.make_task(task, num_envs=n, seed=8), device=DEV)
    b.add_device_event_term("every_step", _push(), "interval", (0.0, 0.0), _vr(ZERO))
    b.add_device_event_term("at_reset", _push(), "reset", None, {"velocity_range": {}})
    gen = torch.Generator(device=DEV).manual_seed(4)
    for t in range(500):
        act = torch.rand((n, 2), device=DEV, generator=gen) * 2 - 1
        oa, ra, ta, ua, _ = a.step(act)
        ob, rb, tb, ub, _ = b.step(act)
        for x, y, what in ((oa["policy"], ob["policy"], "obs"), (ra, rb, "reward"), (ta, tb, "terminated"), (ua, ub, "truncated")):
            assert torch.equal(_bits(x), _bits(y)), f"step {t}: {what}"
    torch.cuda.synchronize()
    assert int(a.sim.episode_length_buf.sum()) > 0 and torch.equal(a.sim.groups, b.sim.groups)


# ---- 4. graph capture -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("task", ["elevation", "drift"])
def test_captured_device_counter_graph_equals_eager_host_counters(task):
    n, K, R = 512, 4, 3
    a, b = _sim(task, n, table=TABLE_8), _sim(task, n, table=TABLE_8)
    gen = torch.Generator(device=DEV).manual_seed(9)
    acts = [torch.rand((n, 2), device=DEV, generator=gen) * 2 - 1 for _ in range(K * R)]
    ref = [tuple(x.clone() for x in a.step_terms(acts[t], t)) for t in range(K * R)]
    outs = [tuple(torch.empty_like(x) for x in ref[0]) for _ in range(K)]
    acts_k = [torch.empty_like(acts[0]) for _ in range(K)]
    stream = torch.cuda.Stream()
    stream.wait_stream(torch.cuda.current_stream())
    g = torch.cuda.CUDAGraph()
    b.set_step_counter(0)
    with torch.cuda.stream(stream), torch.cuda.graph(g, stream=stream):
        for k in range(K):
            b.step_terms(acts_k[k], WheeledSim.device_counter_plus(k), out=outs[k])
        b.advance_counter(K)
    torch.cuda.current_stream().wait_stream(stream)
    b.set_step_counter(0)
    for r in range(R):
        for k in range(K):
            acts_k[k].copy_(acts[r * K + k])
        g.replay()
        torch.cuda.synchronize()
        for k in range(K):
            for x, y in zip(ref[r * K + k], outs[k]):
                assert torch.equal(_bits(x), _bits(y)), f"replay {r} step {k}"
    b.note_device_counter(K * R)
    assert torch.equal(a.groups, b.groups)


def test_calls_that_would_skip_the_events_refuse_the_handle():
    sim = _sim("drift", 64, table=TABLE_1)
    act = torch.zeros((64, 2), device=DEV)
    with pytest.raises(RuntimeError, match="wl_step: the handle has device event terms"):
        sim.step(act, 0)
    with pytest.raises(RuntimeError, match="wl_step_stage_a: the handle has device event terms"):
        sim.step_stage_a(act, 0)
    sim.set_device_events([])
    sim.step(act, 0)                                           # cleared: wl_step runs again
    for bad in ([("interval", (2.0, 1.0), PUSH)], [("reset", None, [(1.0, -1.0)] + PUSH[1:])], [("interval", (-1.0, 1.0), PUSH)],
                [("interval", (0.0, float("nan")), PUSH)], TABLE_8 + TABLE_1):
        with pytest.raises(RuntimeError, match="wl_set_device_events"):
            sim.set_device_events(bad)


# ---- 5. the runner ----------------------------------------------------------------------------------------------------------
T = 8


def _elev_env(n=256, push=True):
    env = ManagerBasedRLEnv(wl.elevation_task(num_envs=n, seed=4), device=DEV)
    if push:
        env.add_device_event_term("push_robot", _push(), "interval", (0.5, 1.5), _vr(PUSH))
    return env


def _runner(env, **kw):
    from wheeledlab_b200.learner import FusedOnPolicyRunner
    from wheeledlab_b200.runs import agent_cfg
    torch.manual_seed(0)
    return FusedOnPolicyRunner(env, agent_cfg("relu", steps=T, save_interval=1), device=DEV, **kw)


def test_runner_trains_the_push_in_one_graph_and_resumes_bit_for_bit(tmp_path):
    from wheeledlab_b200.learner import FusedOnPolicyRunner
    from wheeledlab_b200.runs import agent_cfg
    env_a, env_b, env_p = _elev_env(), _elev_env(), _elev_env(push=False)
    a, b, p = _runner(env_a, log_dir=str(tmp_path)), _runner(env_b), _runner(env_p)
    logs = []
    for r in (a, b, p):
        torch.manual_seed(21)
        logs.append(r.learn(2))
    assert a.it.graph is not None and a.it.roll.device_terms and env_a.common_step_counter == 2 * T
    assert sorted(k for k in logs[0] if k.startswith("Episode_")) == sorted(k for k in logs[2] if k.startswith("Episode_"))
    assert not torch.equal(a.blob, p.blob), "the push is in the rollout"
    c = FusedOnPolicyRunner(env_b, agent_cfg("relu", steps=T, save_interval=1), device=DEV)
    c.load(str(tmp_path / "models" / "model_1.pt"))
    a.alg.state[0] = c.alg.cfg.learning_rate
    for r in (a, c):
        torch.manual_seed(22)
        r.learn(1)
    torch.cuda.synchronize()
    assert env_a.common_step_counter == env_b.common_step_counter == 3 * T
    for name, x, y in (("blob", a.blob, c.blob), ("m", a.alg.m, c.alg.m), ("v", a.alg.v, c.alg.v)):
        assert torch.equal(_bits(x), _bits(y)), name
    assert torch.equal(env_a.sim.groups, env_b.sim.groups)
