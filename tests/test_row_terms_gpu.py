"""Noise, clip and scale on the Elevation and Visual rows on the device (wl_set_row_terms, DESIGN 6r):
- the row kernels equal the CPU twin bit for bit: Elevation at N = 1, 33, 4096 and 8192 with TMA and global-load scans,
  Visual at N = 64 with the camera on, whose camera floats stay those of a handle without row terms; on host and device
  counters, after steps and for observe calls;
- row terms that restate the registered group equal the built-in row over 1000 steps with resets, on both tasks;
- every path writes the modified row: wl_step, wl_step_terms with a device reward term and push, the staged step with a
  Python reward, env.reset / get_observations, step_host; a captured graph of device-counter steps replays to the eager
  host-counter steps;
- the runner trains on the modified row in one graph per iteration and resumes bit for bit, and playback applies the recorded
  row terms;
- the fused act / rollout entries, the pipelined scan and a fan-out refuse or are refused."""
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "tests"))

pytestmark = pytest.mark.gpu

if not torch.cuda.is_available():
    pytest.skip("needs a CUDA device", allow_module_level=True)

import wheeledlab_b200 as wl                                   # noqa: E402
import row_terms_oracle as R                                   # noqa: E402
from wheeledlab_b200 import row_terms                          # noqa: E402
from wheeledlab_b200._lib import WL_ROW_TASK_TERMS, WlError    # noqa: E402
from wheeledlab_b200.env import ManagerBasedRLEnv              # noqa: E402
from wheeledlab_b200.sim import WheeledSim                     # noqa: E402

DEV = "cuda:0"
ELEV_TERMS = [
    ("goal_relative_xyz", ("gaussian", 0.25, 0.5), (-3.0, 7.0), (2.0, -0.5)),
    ("root_euler_xyz", ("uniform", -0.2, 0.6), None, 1.5),
    ("base_lin_vel", ("gaussian", -0.1, 0.3), (-4.0, 2.5), None),
    ("base_ang_vel", None, (-10.0, 10.0), (0.5, 1.0, -2.0)),
    ("last_action", ("uniform", 0.05, 0.15), (-1.0, 1.0), None),
    ("world_height_map", ("uniform", -0.1, 0.3), None, 0.7),
]
ELEV_GAUSS = ELEV_TERMS[:5] + [("world_height_map", ("gaussian", 0.02, 0.05), (-0.3, 0.9), 2.0)]
VIS_TERMS = [("base_lin_vel", ("uniform", -0.1, 0.1), None, (1.0, 2.0, 3.0)),
             ("base_ang_vel", ("gaussian", 0.3, 0.2), (-2.0, 5.0), None),
             ("last_action", ("uniform", -0.1, 0.1), (-1.0, 1.0), 0.5)]


def _spec(task, n, seed=11, corrupt=1, camera="aug"):
    spec = wl.elevation_task(num_envs=n, seed=seed) if task == "elevation" else wl.visual_task(num_envs=n, seed=seed, camera=camera)
    spec.cfg.enable_corruption = corrupt
    return spec


def _sim(spec, terms=None, scan=None):
    sim = WheeledSim(spec, DEV)
    if scan is not None:
        sim.set_scan_tma(scan)
    if terms is not None:
        sim.set_row_terms(terms)
    sim.startup()
    sim.reset(None, 0)
    return sim


def _bits(x):
    return x.contiguous().view(torch.int32).cpu().numpy()


class Twin:
    """The oracle's row under the row terms, from the device state the last call left."""
    def __init__(self, spec):
        self.o = R.RowOracle(spec.cfg, heightfield=spec.heightfield)
        self.o.startup()

    def __call__(self, sim, terms, t, call_idx=-1, base=None):
        self.o.import_state(sim.groups.cpu().numpy())
        obs = None if base is None else np.ascontiguousarray(base.cpu().numpy())
        return self.o.row_observe(terms, t, call_idx, obs=obs).view(np.int32)


# ---- 1. the kernels against the twin --------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [1, 33, 4096, 8192])
@pytest.mark.parametrize("scan", [0, 1])
def test_elevation_kernel_equals_the_twin(n, scan):
    terms = ELEV_TERMS if n % 2 else ELEV_GAUSS
    spec = _spec("elevation", n)
    sim, twin = _sim(spec, terms, scan), Twin(spec)
    steps = 3 if n > 1000 else 12
    for t in range(steps):                                            # host counters, after steps
        obs = sim.step(sim.synth_actions(t), t)[0].clone()
        assert np.array_equal(_bits(obs), twin(sim, terms, t)), (t, n, scan)
    o = sim.observe(steps, 5).clone()                                 # an observe call
    assert np.array_equal(_bits(o), twin(sim, terms, steps, 5))
    sim.set_step_counter(steps)                                       # device counters
    for k in range(2):
        obs = sim.step(sim.synth_actions(steps + k), WheeledSim.device_counter_plus(k))[0].clone()
        assert np.array_equal(_bits(obs), twin(sim, terms, steps + k)), ("device counter", k)
    sim.advance_counter(2)


def test_visual_kernel_equals_the_twin_and_leaves_the_camera_floats():
    n = 64
    spec = _spec("visual", n)
    sim, plain, twin = _sim(spec, VIS_TERMS), _sim(_spec("visual", n)), Twin(spec)
    camf = sim.obs_dim - 8
    assert camf > 0
    for t in range(10):
        act = sim.synth_actions(t)
        obs = sim.step(act, t)[0].clone()
        ref = plain.step(act, t)[0].clone()
        assert np.array_equal(_bits(obs[:, :camf]), _bits(ref[:, :camf])), t
        assert np.array_equal(_bits(obs), twin(sim, VIS_TERMS, t, base=obs)), t
        assert not np.array_equal(_bits(obs[:, camf:]), _bits(ref[:, camf:]))
    o = sim.observe(10, 2).clone()
    assert np.array_equal(_bits(o[:, :camf]), _bits(plain.observe(10, 2)[:, :camf]))
    assert np.array_equal(_bits(o), twin(sim, VIS_TERMS, 10, 2, base=o))
    sim.set_step_counter(10)
    obs = sim.step(sim.synth_actions(10), WheeledSim.device_counter_plus(0))[0].clone()
    assert np.array_equal(_bits(obs), twin(sim, VIS_TERMS, 10, base=obs))


@pytest.mark.parametrize("task", ["elevation", "visual"])
def test_registered_row_terms_are_the_built_in_row_over_1000_steps(task):
    n = 256
    spec = _spec(task, n, corrupt=0, camera=None)
    a, b = _sim(spec), _sim(_spec(task, n, corrupt=0, camera=None), row_terms.registered(task, spec.cfg.obs_clip))
    resets = 0
    for t in range(1000):
        act = a.synth_actions(t)
        oa, _, term, trunc = a.step(act, t)
        ob = b.step(act, t)[0]
        resets += int((term | trunc).sum())
        assert torch.equal(oa.view(torch.int32), ob.view(torch.int32)), t
    assert resets > 0
    assert torch.equal(a.observe(1000, 0).view(torch.int32), b.observe(1000, 0).view(torch.int32))


# ---- 2. every path that writes the row ------------------------------------------------------------------------------------
PUSH = {"velocity_range": {"x": (-0.5, 0.5), "y": (-0.5, 0.5), "yaw": (-1.0, 1.0)}}


def _env(task="elevation", n=128, extra=None, terms=None, seed=5):
    name = "elevation" if task == "elevation" else "visual"
    spec = wl.make_task(name, num_envs=n, seed=seed)
    spec.cfg.enable_corruption = 1
    env = ManagerBasedRLEnv(spec, device=DEV)
    if extra == "device":
        from wheeledlab_b200 import device_terms as dtm
        if str(ROOT / "shims") not in sys.path:
            sys.path.insert(0, str(ROOT / "shims"))
        from isaaclab.envs import mdp
        env.add_device_reward_term("fv", dtm.resolve("forward_vel", dtm.ELEVATION), 0.5)
        env.add_device_event_term("push", mdp.push_by_setting_velocity, "interval", (0.05, 0.2), PUSH)
    elif extra == "python":
        env.add_reward_term("r", lambda e: e.sim.root_pos_w[:, 0], 1.0)
    env.set_row_terms([(f"t{k}", fn, {"noise": nz, "clip": cl, "scale": sc}) for k, (fn, nz, cl, sc) in enumerate(terms or ELEV_TERMS)])
    return env


@pytest.mark.parametrize("extra", [None, "device", "python"])
def test_env_paths_write_the_modified_row(extra):
    env = _env(extra=extra)
    twin = Twin(env.spec)
    obs, _ = env.reset()
    assert np.array_equal(_bits(obs["policy"]), twin(env.sim, ELEV_TERMS, 0, 0))
    for t in range(12):
        obs, *_ = env.step(env.sim.synth_actions(t))
        assert np.array_equal(_bits(obs["policy"]), twin(env.sim, ELEV_TERMS, t)), (extra, t)
    o, _ = env.get_observations()
    assert np.array_equal(_bits(o), twin(env.sim, ELEV_TERMS, 12, 1))
    assert [t[1] for t in env.row_terms] == list(WL_ROW_TASK_TERMS["elevation"])


def test_step_host_writes_the_modified_row():
    for task, terms in (("elevation", ELEV_TERMS), ("visual", VIS_TERMS)):
        env = _env(task, 64, terms=terms)
        twin = Twin(env.spec)
        env.reset()
        for t in range(4):
            obs = env.step_host(env.sim.synth_actions(t).cpu().pin_memory())[0]["policy"]
            torch.cuda.synchronize()
            assert np.array_equal(_bits(obs), twin(env.sim, terms, t, base=obs)), (task, t)


def test_captured_device_counter_graph_equals_eager_host_counters():
    n, K, R = 256, 4, 3
    spec = _spec("elevation", n)
    a, b = _sim(spec, ELEV_GAUSS), _sim(_spec("elevation", n), ELEV_GAUSS)
    gen = torch.Generator(device=DEV).manual_seed(9)
    acts = [torch.rand((n, 2), device=DEV, generator=gen) * 2 - 1 for _ in range(K * R)]
    ref = [a.step(acts[t], t)[0].clone() for t in range(K * R)]
    outs = [(torch.empty((n, 689), device=DEV), torch.empty(n, device=DEV), torch.empty(n, dtype=torch.uint8, device=DEV),
             torch.empty(n, dtype=torch.uint8, device=DEV)) for _ in range(K)]
    acts_k = [torch.empty_like(acts[0]) for _ in range(K)]
    stream = torch.cuda.Stream()
    stream.wait_stream(torch.cuda.current_stream())
    g = torch.cuda.CUDAGraph()
    b.set_step_counter(0)
    with torch.cuda.stream(stream), torch.cuda.graph(g, stream=stream):
        for k in range(K):
            b.step(acts_k[k], WheeledSim.device_counter_plus(k), out=outs[k])
        b.advance_counter(K)
    torch.cuda.current_stream().wait_stream(stream)
    b.set_step_counter(0)
    for r in range(R):
        for k in range(K):
            acts_k[k].copy_(acts[r * K + k])
        g.replay()
        torch.cuda.synchronize()
        for k in range(K):
            assert torch.equal(ref[r * K + k].view(torch.int32), outs[k][0].view(torch.int32)), f"replay {r} step {k}"


# ---- 3. training and playback -----------------------------------------------------------------------------------------------
T = 8


def _runner(env, **kw):
    from wheeledlab_b200.learner import FusedOnPolicyRunner
    from wheeledlab_b200.runs import agent_cfg
    torch.manual_seed(0)
    return FusedOnPolicyRunner(env, agent_cfg("relu", steps=T, save_interval=1), device=DEV, **kw)


@pytest.mark.parametrize("task,n", [("elevation", 4096), ("visual", 64)])
def test_runner_trains_on_the_modified_row_in_one_graph_and_resumes_bit_for_bit(tmp_path, task, n):
    terms = ELEV_GAUSS if task == "elevation" else VIS_TERMS
    env_a, env_b = _env(task, n, terms=terms), _env(task, n, terms=terms)
    a, b = _runner(env_a, log_dir=str(tmp_path)), _runner(env_b)
    assert a.it.roll.rows
    for r in (a, b):
        torch.manual_seed(21)
        r.learn(2)
    assert a.it.graph is not None and env_a.common_step_counter == 2 * T
    twin = Twin(env_a.spec)
    last = a.it.roll.slab.obs[T - 1]
    assert np.array_equal(_bits(last), twin(env_a.sim, terms, 2 * T - 1, base=last)), "the slab holds the modified row"
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


def test_playback_applies_the_recorded_row_terms(tmp_path):
    sys.path.insert(0, str(ROOT / "tools"))
    import play_policy
    from wheeledlab_b200.policy import actor_mean
    from wheeledlab_b200.runs import agent_cfg, save_run_config
    env = _env("elevation", 128, terms=ELEV_GAUSS)
    r = _runner(env, log_dir=str(tmp_path))
    r.learn(1)
    pol = r.get_inference_policy()
    obs, _ = env.get_observations()
    assert torch.equal(pol(obs), actor_mean(r.blob, 689, obs, "relu"))
    save_run_config(str(tmp_path), "Isaac-MushrElevationRL-v0", 128, 5, agent_cfg("relu", steps=T, save_interval=1), row_terms=env.row_terms)
    assert play_policy.main(["-p", str(tmp_path), "--steps", "16"]) == 0
    res = play_policy.resolve(play_policy.parser().parse_args(["-p", str(tmp_path), "--steps", "16"]))
    runner, roll, _ = play_policy.play(res, 16)
    assert roll.sim.row_terms == 6 and roll.rows and np.array_equal(_bits(runner.blob), _bits(r.blob))


# ---- 4. refusals -----------------------------------------------------------------------------------------------------------
def test_the_fused_entries_the_pipelined_scan_and_a_fan_out_refuse():
    import ctypes as C
    from wheeledlab_b200._lib import WlPolicyOut, lib
    vis = _sim(_spec("visual", 64, camera=None), VIS_TERMS)
    p = lambda x: C.c_void_p(x.data_ptr())
    obs, blob = torch.zeros((64, 8), device=DEV), torch.zeros(8192, device=DEV)
    f, u = torch.zeros(64 * 4, device=DEV), torch.zeros(64, dtype=torch.uint8, device=DEV)
    out = WlPolicyOut(p(f), p(f), p(f), p(f))
    assert lib.wl_act_step(vis._h, p(obs), p(blob), out, p(obs), p(f), p(u), p(u), None, 0, None) == -3
    assert b"row terms" in lib.wl_last_error()
    assert lib.wl_act_infer_step(vis._h, p(obs), p(blob), p(f), p(obs), p(f), p(u), p(u), None, 0, None) == -3
    assert b"row terms" in lib.wl_last_error()
    assert lib.wl_rollout(vis._h, 2, None, None, p(obs), p(f), p(u), p(u), p(f), 0, None) == -3
    assert b"row terms" in lib.wl_last_error()
    with pytest.raises(WlError):
        vis.set_peer_fanout([16])                                   # (the fan-out is the Drift step kernel's)
    elev = _sim(_spec("elevation", 16), ELEV_TERMS)
    with pytest.raises(WlError, match="row-terms variant"):
        elev.set_scan_tma(2)
    elev.set_row_terms([])
    elev.set_scan_tma(2)
    with pytest.raises(WlError, match="row-terms variant"):
        elev.set_row_terms(ELEV_TERMS)
    assert elev.row_terms == 0
    for bad in (ELEV_TERMS[:5], [ELEV_TERMS[1]] + ELEV_TERMS[1:], ELEV_TERMS[:5] + [("world_height_map", None, None, (1.0, 2.0))],
                ELEV_TERMS[:4] + [("last_action", ("gaussian", 0.0, float("nan")), None, None), ELEV_TERMS[5]]):
        with pytest.raises(WlError):
            _sim(_spec("elevation", 4)).set_row_terms(bad)
    drift = WheeledSim(wl.make_task("drift", num_envs=16), DEV)
    with pytest.raises(WlError, match="Drift family"):
        drift.set_row_terms(VIS_TERMS)
    with pytest.raises(WlError, match="call_idx"):
        vis.observe(0, 1 << 23)
