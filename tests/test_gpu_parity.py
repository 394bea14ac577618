"""GPU parity tests: the CUDA path (through the C-ABI) against the CPU oracle on the same seeded inputs.
Bit-exact for every output (the arithmetic contract makes fp32 results identical), including done masks
and reset indices, over trajectories long enough to contain many auto-resets."""
import ctypes as C
from pathlib import Path

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
import oracle_lib as O  # noqa: E402


def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


def _pair(n, seed=42, **kw):
    import wheeledlab_b200 as wl
    spec = wl.drift_task(num_envs=n, seed=seed, **kw)
    sim = wl.WheeledSim(spec, "cuda:0")
    sim.startup(); sim.reset(None, 0)
    orc = O.Oracle(spec.cfg)
    orc.startup(); orc.reset(None, 0)
    return spec, sim, orc


def _state_groups(sim):
    return sim.groups.detach().cpu().numpy()


def test_loaded_native_library_is_in_tree():
    _need_gpu()
    import wheeledlab_b200 as wl
    maps = open("/proc/self/maps").read()
    assert str(wl.LIB_PATH) in maps


def test_detmath_bit_exact():
    _need_gpu()
    import wheeledlab_b200 as wl
    rng = np.random.default_rng(0)
    cases = {0: rng.uniform(-8, 8, 100000), 1: rng.uniform(-8, 8, 100000), 2: rng.normal(0, 10, 100000),
             4: rng.uniform(1e-7, 1, 100000), 5: rng.uniform(-0.6, 0.6, 100000), 6: rng.uniform(-1, 1, 100000),
             7: -rng.uniform(0, 90, 100000)}
    for op, x in cases.items():
        x = x.astype(np.float32)
        d_in = torch.from_numpy(x).cuda(); d_out = torch.empty_like(d_in)
        wl._lib.check(wl.lib.wl_test_detmath(op, d_in.data_ptr(), d_in.data_ptr(), d_out.data_ptr(), x.size, None))
        torch.cuda.synchronize()
        assert np.array_equal(_bits(d_out.cpu().numpy()), _bits(O.detmath(op, x))), f"op {op}"
    x, y = rng.normal(size=100000).astype(np.float32), rng.normal(size=100000).astype(np.float32)
    dx, dy = torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda(); d_out = torch.empty_like(dx)
    wl._lib.check(wl.lib.wl_test_detmath(3, dx.data_ptr(), dy.data_ptr(), d_out.data_ptr(), x.size, None))
    torch.cuda.synchronize()
    assert np.array_equal(_bits(d_out.cpu().numpy()), _bits(O.detmath(3, x, y)))


def test_philox_bit_exact_and_kat():
    _need_gpu()
    import wheeledlab_b200 as wl
    out = torch.empty((1000, 4), dtype=torch.int32, device="cuda")
    wl._lib.check(wl.lib.wl_test_philox(1234567890123, 17, 3, 5, 7, out.data_ptr(), 1000, None))
    torch.cuda.synchronize()
    assert np.array_equal(out.cpu().numpy().view(np.uint32), O.philox(1234567890123, 17, 3, 5, 7, 1000))
    wl._lib.check(wl.lib.wl_test_philox(0, 0, 0, 0, 0, out.data_ptr(), 1, None))
    torch.cuda.synchronize()
    assert [hex(x) for x in out[0].cpu().numpy().view(np.uint32)] == ["0x6627e8d5", "0xe169c58d", "0xbc57ac4c", "0x9b00dbd8"]


def test_startup_and_reset_state_bit_exact():
    _need_gpu()
    spec, sim, orc = _pair(1000, seed=9)
    torch.cuda.synchronize()
    assert np.array_equal(_bits(_state_groups(sim)), _bits(orc.export_state()))
    ids = np.array([3, 999, 17, 500], np.int64)
    sim.reset(torch.from_numpy(ids).cuda(), 77); orc.reset(ids, 77)
    torch.cuda.synchronize()
    assert np.array_equal(_bits(_state_groups(sim)), _bits(orc.export_state()))


@pytest.mark.parametrize("variant", [1, 4, 8])   # one thread per env / four lanes (one per wheel) per env / quad + aux warp
@pytest.mark.parametrize("n,steps,kw", [
    (256, 1000, {}),                               # RSS_DRIFT settings, DR + pushes + noise on
    (333, 300, {"randomize": False}),              # ragged N (not a multiple of the CTA), DR off
    (64, 300, {"drive": "4wd"}),                   # BASELINE config 4: 4WD action map + 4 driven wheels
    (1, 260, {}),                                  # single env (BASELINE config 1 plumbing size)
])
def test_step_trajectory_bit_exact(n, steps, kw, variant):
    """1000-step trajectories: obs, reward, done masks, episode log and the full state, every step."""
    _need_gpu()
    spec, sim, orc = _pair(n, seed=42, **kw)
    sim.set_kernel_variant(variant)
    n_done = 0
    for t in range(steps):
        act = sim.synth_actions(t, dist=t % 2)
        a_np = act.cpu().numpy()
        assert np.array_equal(_bits(a_np), _bits(orc.synth_actions(t, dist=t % 2)))
        log = torch.empty(16, device="cuda")
        obs, rew, term, trunc = sim.step(act, t, log=log)
        sim.flush_log()                                  # the row of step t is published by the next launch on the handle
        o_obs, o_rew, o_term, o_trunc = orc.step(a_np, t)
        torch.cuda.synchronize()
        assert np.array_equal(term.cpu().numpy(), o_term), f"terminated mask differs at step {t}"
        assert np.array_equal(trunc.cpu().numpy(), o_trunc), f"time-out mask differs at step {t}"
        assert np.array_equal(_bits(rew.cpu().numpy()), _bits(o_rew)), f"reward differs at step {t}"
        assert np.array_equal(_bits(obs.cpu().numpy()), _bits(o_obs)), f"obs differs at step {t}"
        n_done += int((o_term | o_trunc).sum())
        lg, got = orc.log(), log.cpu().numpy()
        assert np.allclose(got[:8], lg[:8], rtol=1e-5, atol=1e-4)          # float atomics: order-dependent sum
        assert np.array_equal(got[8:11], lg[8:11].astype(np.float32))
        if t % 50 == 0 or t == steps - 1:
            assert np.array_equal(_bits(_state_groups(sim)), _bits(orc.export_state())), f"state differs at step {t}"
    assert n_done >= n, "trajectory too short to exercise auto-reset"


def test_relative_l2_over_1000_steps_is_zero():
    """north_star: state trajectories within 1e-3 relative L2 over 1000 steps (here: exactly 0)."""
    _need_gpu()
    spec, sim, orc = _pair(128, seed=1)
    num = den = 0.0
    for t in range(1000):
        act = sim.synth_actions(t)
        sim.step(act, t); orc.step(act.cpu().numpy(), t)
        if t % 100 == 99:
            a, b = _state_groups(sim)[:6].astype(np.float64), orc.export_state()[:6].astype(np.float64)
            a[0, :, 3] = b[0, :, 3] = 0          # int bits (episode length) excluded from the float norm
            num += ((a - b) ** 2).sum(); den += (b ** 2).sum()
    assert (num / den) ** 0.5 <= 1e-3 and num == 0.0


def test_observe_resamples_noise_bit_exact():
    _need_gpu()
    spec, sim, orc = _pair(200, seed=4)
    a = sim.observe(0, 0).cpu().numpy(); b = sim.observe(0, 1).cpu().numpy()
    assert np.array_equal(_bits(a), _bits(orc.observe(0, 0))) and np.array_equal(_bits(b), _bits(orc.observe(0, 1)))
    assert not np.array_equal(a[:, :12], b[:, :12]) and np.array_equal(a[:, 12:], b[:, 12:])


def test_kernel_variants_agree_at_full_size():
    """4096 envs (RSS_DRIFT_CONFIG size): thread-per-env and quad-per-env kernels give identical bits."""
    _need_gpu()
    import wheeledlab_b200 as wl
    a = wl.WheeledSim(wl.drift_task(num_envs=4096, seed=42), "cuda:0"); b = wl.WheeledSim(wl.drift_task(num_envs=4096, seed=42), "cuda:0")
    d = wl.WheeledSim(wl.drift_task(num_envs=4096, seed=42), "cuda:0")
    a.set_kernel_variant(1); b.set_kernel_variant(4); d.set_kernel_variant(8)
    for s in (a, b, d):
        s.startup(); s.reset(None, 0)
    for t in range(400):
        act = a.synth_actions(t)
        ra, rb, rd = a.step(act, t), b.step(act, t), d.step(act, t)
        for x, y, z in zip(ra, rb, rd):
            assert torch.equal(x, y) and torch.equal(x, z), f"variant mismatch at step {t}"
    assert torch.equal(a.groups, b.groups) and torch.equal(a.groups, d.groups) and torch.equal(a.rew_weight, d.rew_weight)


def test_sharding_invariance_two_shards_equal_one():
    """BASELINE config 5 property: envs keyed by GLOBAL id => concat of shards == one big run, bit for bit."""
    _need_gpu()
    import wheeledlab_b200 as wl
    n, steps = 512, 300
    whole = wl.WheeledSim(wl.drift_task(num_envs=n, seed=21), "cuda:0")
    lo = wl.WheeledSim(wl.drift_task(num_envs=n // 2, seed=21, env_id_offset=0), "cuda:0")
    hi = wl.WheeledSim(wl.drift_task(num_envs=n // 2, seed=21, env_id_offset=n // 2), "cuda:0")
    for s in (whole, lo, hi):
        s.startup(); s.reset(None, 0)
    for t in range(steps):
        aw = whole.synth_actions(t)
        ow = whole.step(aw, t)
        ol = lo.step(lo.synth_actions(t), t); oh = hi.step(hi.synth_actions(t), t)
        for w, l, h in zip(ow, ol, oh):
            assert torch.equal(w, torch.cat([l, h], dim=0)), f"shard mismatch at step {t}"
    assert torch.equal(whole.groups, torch.cat([lo.groups, hi.groups], dim=1))


def test_curriculum_on_device_matches_oracle():
    """increase_reward_weight_over_time evaluated by the step kernel's last CTA: fires only at episode boundaries of the
    global counter AND only if some env reset in that step; weights and subsequent rewards match the oracle."""
    _need_gpu()
    import wheeledlab_b200 as wl
    spec = wl.drift_task(num_envs=64, seed=2)
    spec.cfg.curr_every[0] = 1                       # term 0 (side_slip += 20) every episode, term 2 every 2nd
    spec.cfg.curr_every[2] = 2
    sim = wl.WheeledSim(spec, "cuda:0"); sim.startup(); sim.reset(None, 0)
    orc = O.Oracle(spec.cfg); orc.startup(); orc.reset(None, 0)
    w0 = sim.rew_weight.cpu().numpy().copy()
    exp = w0.copy()
    fired = 0
    for t in range(0, 1002):
        act = sim.synth_actions(t)
        _, rew, _, _ = sim.step(act, t); _, o_rew, _, _ = orc.step(act.cpu().numpy(), t)
        assert np.array_equal(_bits(rew.cpu().numpy()), _bits(o_rew)), t
        if (t + 1) % 250 == 0:                       # episode boundary of the GLOBAL counter
            E = (t + 1) // 250
            if orc.any_reset():                      # the reference only evaluates the terms when >= 1 env reset this step
                exp[0] += 20.0                       # every episode
                if (E + 1) % 2 == 0:
                    exp[6] += -1000.0                # every 2nd episode
                fired += 1
            w = sim.rew_weight.cpu().numpy()
            assert np.array_equal(w, orc.weights()) and np.array_equal(w, exp), (t, w, exp)
        elif t % 97 == 0:
            assert np.array_equal(sim.rew_weight.cpu().numpy(), exp), t      # never changes off-boundary
    assert fired >= 1


def test_device_counter_graph_replay_equals_host_counter():
    """wl_step on the device-resident counter (base + 0, then base += 1) captured ONCE in a CUDA graph and replayed T times ==
    T host-counter steps."""
    _need_gpu()
    import wheeledlab_b200 as wl
    n, T = 512, 300
    a = wl.WheeledSim(wl.drift_task(num_envs=n, seed=6), "cuda:0"); b = wl.WheeledSim(wl.drift_task(num_envs=n, seed=6), "cuda:0")
    for s_ in (a, b):
        s_.startup(); s_.reset(None, 0)
    act = torch.empty((n, 2), device="cuda"); out = tuple(torch.empty_like(x) for x in a.step(a.synth_actions(0), 0))
    b.step(b.synth_actions(0), 0)                    # both are at counter 1 now
    b.set_step_counter(1)
    stream = torch.cuda.Stream(); stream.wait_stream(torch.cuda.current_stream())
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(stream):
        with torch.cuda.graph(g, stream=stream):
            b.synth_actions(wl.WheeledSim.DEVICE_COUNTER, out=act)
            b.step(act, wl.WheeledSim.DEVICE_COUNTER, out=out)
            b.advance_counter(1)
    torch.cuda.current_stream().wait_stream(stream)
    b.set_step_counter(1)                            # capture moved the host mirror of the counter; nothing has run yet
    for t in range(1, T):
        ref = a.step(a.synth_actions(t), t)
        g.replay()
        torch.cuda.synchronize()
        for x, y in zip(ref, out):
            assert torch.equal(x, y), f"graph replay differs at step {t}"
    b.note_device_counter(T)
    assert torch.equal(a.groups, b.groups) and torch.equal(a.rew_weight, b.rew_weight)


def test_env_api_surface_and_full_size_properties():
    """RSS_DRIFT_CONFIG size (4096 envs): ManagerBasedRLEnv surface + size-independent properties."""
    _need_gpu()
    import wheeledlab_b200 as wl
    env = wl.make("Isaac-MushrDriftRL-v0", num_envs=4096, seed=42)
    obs, extras = env.reset()
    assert obs["policy"].shape == (4096, 14) and env.max_episode_length == 250 and env.num_envs == 4096
    assert env.action_manager.total_action_dim == 2 and env.observation_manager.group_obs_dim["policy"] == (14,)
    total_done = torch.zeros((), device="cuda")
    prev_len = env.episode_length_buf.clone()
    for t in range(300):
        a = env.sim.synth_actions(t)
        obs, rew, term, trunc, extras = env.step(a)
        assert term.dtype == torch.bool and trunc.dtype == torch.bool and rew.shape == (4096,)
        done = term | trunc
        ep = env.episode_length_buf
        # reset indices: episode length is 0 exactly where done, else previous + 1
        assert torch.equal(ep == 0, done)
        assert torch.equal(ep[~done], prev_len[~done] + 1)
        # a reset env has zero velocity (before pushes) only approximately -> check pose is on the track & upright
        q = env.scene["robot"].data.root_quat_w
        assert torch.allclose((q * q).sum(-1), torch.ones(4096, device="cuda"), atol=1e-5)
        assert torch.isfinite(obs["policy"]).all() and torch.isfinite(rew).all()
        assert "Episode_Reward/side_slip" in extras["log"] and extras["log"]["Episode_Termination/time_out"].shape == ()
        total_done += done.sum(); prev_len = ep.clone()
    assert total_done.item() >= 4096
    assert (env.episode_length_buf < 250).all()
    tc = env.reward_manager.get_term_cfg("side_slip"); tc.weight += 5; env.reward_manager.set_term_cfg("side_slip", tc)
    assert env.reward_manager.get_term_cfg("side_slip").weight == tc.weight
    o1, _ = env.get_observations(); o2, _ = env.get_observations()
    assert not torch.equal(o1, o2)            # noise is re-sampled (SURVEY 3.4)
    env.close()


def test_cuda_graph_replay_matches_eager():
    _need_gpu()
    import wheeledlab_b200 as wl
    n, k = 1024, 16
    a = wl.WheeledSim(wl.drift_task(num_envs=n, seed=8), "cuda:0"); b = wl.WheeledSim(wl.drift_task(num_envs=n, seed=8), "cuda:0")
    for s in (a, b):
        s.startup(); s.reset(None, 0)
    acts = torch.stack([a.synth_actions(t) for t in range(k)])
    outs_a = [tuple(x.clone() for x in a.step(acts[t], t)) for t in range(k)]
    bufs = [tuple(torch.empty_like(x) for x in outs_a[0]) for _ in range(k)]
    stream = torch.cuda.Stream()
    stream.wait_stream(torch.cuda.current_stream())
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(stream):
        with torch.cuda.graph(g, stream=stream):
            for t in range(k):
                b.step(acts[t], t, out=bufs[t])
    g.replay(); torch.cuda.synchronize()
    for t in range(k):
        for x, y in zip(outs_a[t], bufs[t]):
            assert torch.equal(x, y)
    assert torch.equal(a.groups, b.groups)


# ---------------------------------------------------------------------------------------------------------------
# Elevation task (BASELINE config 3): height-field contact, goal command, 26x26 TMA-staged ray-cast observation
# ---------------------------------------------------------------------------------------------------------------
def _elev_pair(n, seed=42):
    import wheeledlab_b200 as wl
    spec = wl.elevation_task(num_envs=n, seed=seed)
    sim = wl.WheeledSim(spec, "cuda:0")
    sim.startup(); sim.reset(None, 0)
    orc = O.Oracle(spec.cfg, heightfield=spec.heightfield)
    orc.startup(); orc.reset(None, 0)
    return spec, sim, orc


def test_scan_pipeline_walks_several_envs_per_cta():
    """The pipelined ray-caster runs min(N, 132 x 6 = 792) persistent CTAs on the H100: with more envs than that CTAs re-use their two stages
    (mbarrier phases flip), and the rows must still equal the oracle's and the plain-load kernel's bit for bit."""
    _need_gpu()
    n = 4000
    spec, sim, orc = _elev_pair(n)
    for t in range(3):
        act = sim.synth_actions(t)
        sim.set_scan_tma(2); sim.step(act, t)
        o_obs = orc.step(act.cpu().numpy(), t)[0]
    a2 = sim.observe(3).cpu().numpy()
    sim.set_scan_tma(0); a0 = sim.observe(3).cpu().numpy()
    sim.set_scan_tma(1); a1 = sim.observe(3).cpu().numpy()
    ref = orc.observe(3)
    assert np.array_equal(_bits(a2), _bits(ref)) and np.array_equal(_bits(a0), _bits(ref)) and np.array_equal(_bits(a1), _bits(ref))


@pytest.mark.parametrize("variant,tma", [(1, 2), (4, 2), (4, 1), (4, 0)])
def test_elevation_trajectory_bit_exact(variant, tma):
    _need_gpu()
    n, steps = 96, 260
    spec, sim, orc = _elev_pair(n)
    sim.set_kernel_variant(variant); sim.set_scan_tma(tma)
    assert sim.obs_dim == 689
    a0 = sim.observe(0).cpu().numpy()
    assert np.array_equal(_bits(a0), _bits(orc.observe(0)))
    counts = np.zeros(5)
    for t in range(steps):
        act = sim.synth_actions(t)
        log = torch.empty(16, device="cuda")
        obs, rew, term, trunc = sim.step(act, t, log=log)
        sim.flush_log()
        o_obs, o_rew, o_term, o_trunc = orc.step(act.cpu().numpy(), t)
        torch.cuda.synchronize()
        assert np.array_equal(term.cpu().numpy(), o_term) and np.array_equal(trunc.cpu().numpy(), o_trunc), t
        assert np.array_equal(_bits(rew.cpu().numpy()), _bits(o_rew)), f"reward differs at step {t}"
        got = obs.cpu().numpy()
        assert np.array_equal(_bits(got[:, :13]), _bits(o_obs[:, :13])), f"proprio obs differs at step {t}"
        assert np.array_equal(_bits(got[:, 13:]), _bits(o_obs[:, 13:])), f"height scan differs at step {t}"
        lg = orc.log(); counts += lg[9:14]
        assert np.array_equal(log.cpu().numpy()[8:14], lg[8:14].astype(np.float32))
        if t % 65 == 0 or t == steps - 1:
            assert np.array_equal(_bits(_state_groups(sim)), _bits(orc.export_state())), f"state differs at step {t}"
    assert counts[0] > 0 and counts[2] > 0 and counts.sum() >= n        # time-outs, stuck, ... all exercised
    sc = got[:, 13:]
    assert sc.max() <= 10 and sc.min() >= -10 and (np.abs(sc) < 9.9).mean() > 0.5


def test_elevation_full_size_properties():
    """RSS_ELEV_CONFIG size (4096 envs): env surface, obs width 689, scan/clip bounds, reset semantics."""
    _need_gpu()
    import wheeledlab_b200 as wl
    env = wl.make("Isaac-MushrElevationRL-v0", num_envs=4096, seed=42)
    obs, _ = env.reset()
    assert obs["policy"].shape == (4096, 689) and env.max_episode_length == 200
    prev = env.episode_length_buf.clone()
    for t in range(60):
        obs, rew, term, trunc, extras = env.step(env.sim.synth_actions(t))
        done = term | trunc
        ep = env.episode_length_buf
        assert torch.equal(ep == 0, done) and torch.equal(ep[~done], prev[~done] + 1)
        o = obs["policy"]
        assert torch.isfinite(o).all() and o[:, 5:].abs().max() <= 10.0
        z = env.scene["robot"].data.root_pos_w[:, 2]
        assert torch.allclose(z[done], torch.full_like(z[done], 0.25))          # respawn at default root z (:147-149)
        prev = ep.clone()
    assert "Episode_Termination/stuck" in extras["log"] and env.command_manager.get_command("goal_pose").shape == (4096, 4)
    env.close()


def test_step_host_matches_device_step():
    """wl_step_host (host buffers in/out, one C call) == wl_step on device tensors, bit for bit."""
    _need_gpu()
    import wheeledlab_b200 as wl
    a = wl.make("Isaac-MushrDriftRL-v0", num_envs=512, seed=3); b = wl.make("Isaac-MushrDriftRL-v0", num_envs=512, seed=3)
    a.reset(); b.reset()
    h_in = b.host_action_buffer
    assert h_in.is_pinned()
    pinned_block = torch.empty((40, 512, 2)).pin_memory()
    pinned_rows = [pinned_block[t] for t in range(40)]
    for t in range(40):
        b.host_transport = "zero_copy" if (t // 4) % 2 else "copy"      # every input kind under both transports
        act = a.sim.synth_actions(t)
        pinned_rows[t].copy_(act.cpu())
        oa, ra, ta, ua, _ = a.step(act)
        if t % 4 < 2:
            h_in.copy_(act.cpu())
            ob, rb, tb, ub, ex = b.step_host(h_in)                       # the env's own pinned buffer
        elif t % 4 == 2:
            ob, rb, tb, ub, ex = b.step_host(pinned_rows[t])             # a pinned block of the caller: read in place
        else:
            ob, rb, tb, ub, ex = b.step_host(act.cpu())                  # pageable memory: staged through the env's buffer
        assert rb.device.type == "cpu" and tb.dtype == torch.bool
        assert torch.equal(oa["policy"], ob["policy"]) and torch.equal(ra.cpu(), rb) and torch.equal(ta.cpu(), tb) and torch.equal(ua.cpu(), ub)
        assert float(ex["log"]["Episode_Termination/time_out"]) >= 0
    assert torch.equal(a.sim.groups, b.sim.groups)


# ---------------------------------------------------------------------------------------------------------------
# Visual task, physics side (traversability-map reward, out-of-map termination, random traversable respawn)
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("variant", [1, 4])
def test_visual_trajectory_bit_exact(variant):
    _need_gpu()
    import wheeledlab_b200 as wl
    n, steps = 128, 120
    spec = wl.visual_task(num_envs=n, seed=42)
    sim = wl.WheeledSim(spec, "cuda:0"); sim.set_kernel_variant(variant)
    sim.startup(); sim.reset(None, 0)
    orc = O.Oracle(spec.cfg, heightfield=spec.heightfield); orc.startup(); orc.reset(None, 0)
    assert sim.obs_dim == 8
    assert np.array_equal(_bits(sim.observe(0).cpu().numpy()), _bits(orc.observe(0)))
    n_done = 0
    for t in range(steps):
        act = sim.synth_actions(t)
        obs, rew, term, trunc = sim.step(act, t)
        o_obs, o_rew, o_term, o_trunc = orc.step(act.cpu().numpy(), t)
        torch.cuda.synchronize()
        assert np.array_equal(term.cpu().numpy(), o_term) and np.array_equal(trunc.cpu().numpy(), o_trunc), t
        assert np.array_equal(_bits(rew.cpu().numpy()), _bits(o_rew)) and np.array_equal(_bits(obs.cpu().numpy()), _bits(o_obs)), t
        n_done += int((o_term | o_trunc).sum())
    assert np.array_equal(_bits(_state_groups(sim)), _bits(orc.export_state())) and n_done >= 2 * n
    env = wl.make("Isaac-MushrVisualRL-v0", num_envs=64)
    o, _ = env.reset()
    assert o["policy"].shape == (64, 3208) and env.max_episode_length == 50      # registered task: camera + 8 proprio floats
    env = wl.ManagerBasedRLEnv(wl.visual_task(num_envs=64), device="cuda:0")
    assert env.reset()[0]["policy"].shape == (64, 8)


def test_articulation_views_and_suspension():
    """env.scene["robot"].data.* (IsaacLab names): zero-copy root state, derived joint state incl. suspension.  A smoke check;
    tests/test_articulation_cpu.py and tests/test_articulation_gpu.py are the tests of record for these views."""
    _need_gpu()
    import wheeledlab_b200 as wl
    env = wl.make("Isaac-MushrDriftRL-v0", num_envs=256, seed=1)
    env.reset()
    for t in range(30):
        env.step(env.sim.synth_actions(t))
    d = env.scene["robot"].data
    jp, jv = d.joint_pos, d.joint_vel
    assert jp.shape == (256, 10) and jv.shape == (256, 10)
    susp = jp[:, 6:10]
    assert susp.abs().max() <= 0.01 + 1e-6 and (susp > 0.001).float().mean() > 0.9      # ~3.7 mm static deflection, +-10 mm travel
    ids, names = env.scene["robot"].find_joints(".*_steer")
    assert names == ["front_left_wheel_steer", "front_right_wheel_steer"] and torch.equal(jp[:, ids], env.sim.steer_pos)
    # write_root_pose_to_sim goes through the zero-copy views (events.py:132-133)
    pose = torch.tensor([[0.8, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0]], device="cuda").repeat(4, 1)
    env.scene["robot"].write_root_pose_to_sim(pose, env_ids=torch.tensor([0, 5, 7, 9], device="cuda"))
    assert torch.equal(d.root_pos_w[[0, 5, 7, 9]], pose[:, :3]) and torch.equal(d.root_quat_w[5], pose[0, 3:])
    vb = d.root_lin_vel_b
    assert vb.shape == (256, 3) and torch.isfinite(vb).all()


def test_graphed_policy_rollout_equals_eager_loop():
    """T x (MLP policy -> env.step) captured in one CUDA graph == the same loop run eagerly with host counters."""
    _need_gpu()
    import wheeledlab_b200 as wl
    from wheeledlab_b200.rollout import GraphedRollout
    n, T = 1024, 64
    torch.manual_seed(0)
    mlp = torch.nn.Sequential(torch.nn.Linear(14, 64), torch.nn.ELU(), torch.nn.Linear(64, 64), torch.nn.ELU(), torch.nn.Linear(64, 2)).cuda()
    policy = lambda obs: mlp(obs)
    a = wl.WheeledSim(wl.drift_task(num_envs=n, seed=9), "cuda:0"); b = wl.WheeledSim(wl.drift_task(num_envs=n, seed=9), "cuda:0")
    for s_ in (a, b):
        s_.startup(); s_.reset(None, 0)
    with torch.no_grad():
        roll = GraphedRollout(b, policy, T).capture(step_counter=0)
        for it in range(3):
            slab = roll.run()
            torch.cuda.synchronize()
            obs = a.observe(0, 0) if it == 0 else obs
            for k in range(T):
                act = policy(obs).contiguous()
                obs, rew, term, trunc = a.step(act, it * T + k)
                assert torch.equal(slab.obs[k], obs) and torch.equal(slab.rewards[k], rew), (it, k)
                assert torch.equal(slab.terminated[k], term) and torch.equal(slab.truncated[k], trunc)
    assert torch.equal(a.groups, b.groups)


def test_fused_k_step_rollout_equals_k_single_steps():
    """wl_rollout (K env.steps in one launch, state in registers, in-kernel actions) == K x (synth_actions + wl_step)."""
    _need_gpu()
    import wheeledlab_b200 as wl
    from wheeledlab_b200.distributed import RolloutSlab
    n, K = 700, 100
    a = wl.WheeledSim(wl.drift_task(num_envs=n, seed=13), "cuda:0"); b = wl.WheeledSim(wl.drift_task(num_envs=n, seed=13), "cuda:0")
    for s_ in (a, b):
        s_.startup(); s_.reset(None, 0)
    slab = RolloutSlab(K, n, 14, 2, "cuda:0"); logs = torch.empty((K, 16), device="cuda")
    for it, t0 in enumerate((0, 100, 200)):          # 200..299 crosses counter 250 -> must be split
        if t0 == 200:
            with pytest.raises(wl.WlError):
                b.rollout(K, t0, slab, logs)
            b.rollout(50, 200, slab, logs); first = [x[:50].clone() for x in (slab.obs, slab.rewards, slab.terminated, slab.truncated, slab.actions)]
            b.rollout(50, 250, slab, logs)
            got = [torch.cat([f, x[:50]]) for f, x in zip(first, (slab.obs, slab.rewards, slab.terminated, slab.truncated, slab.actions))]
        else:
            b.rollout(K, t0, slab, logs)
            got = [x.clone() for x in (slab.obs, slab.rewards, slab.terminated, slab.truncated, slab.actions)]
        for k in range(K):
            act = a.synth_actions(t0 + k)
            log = torch.empty(16, device="cuda")
            obs, rew, term, trunc = a.step(act, t0 + k, log=log); a.flush_log()
            assert torch.equal(got[4][k], act) and torch.equal(got[0][k], obs) and torch.equal(got[1][k], rew), (t0, k)
            assert torch.equal(got[2][k], term) and torch.equal(got[3][k], trunc)
            if t0 != 200:
                assert torch.allclose(logs[k], log, rtol=1e-5, atol=1e-4) and torch.equal(logs[k, 8:], log[8:])
        assert torch.equal(a.groups, b.groups) and torch.equal(a.rew_weight, b.rew_weight)


def test_gae_matches_rsl_rl_formula():
    """wl_gae vs a torch fp32 restatement of rsl_rl's compute_returns (+ time-out bootstrap), tolerance 1e-5."""
    _need_gpu()
    from wheeledlab_b200.learner import compute_returns
    torch.manual_seed(0)
    for T, N in ((128, 4096), (100, 1000), (256, 64), (24, 8192), (300, 512), (5, 33), (1, 1)):   # segment-parallel (T <= 256) and streaming scans
        rew = torch.randn(T, N, device="cuda"); val = torch.randn(T, N, device="cuda"); last = torch.randn(N, device="cuda")
        done = torch.rand(T, N, device="cuda") < 0.05
        tout = done & (torch.rand(T, N, device="cuda") < 0.5)
        gamma, lam = 0.99, 0.95
        ret, adv = compute_returns(rew, val, last, done, gamma, lam, time_outs=tout)
        r2 = rew + gamma * val * tout.float()
        a = torch.zeros(N, device="cuda"); exp_ret = torch.empty_like(rew)
        for t in reversed(range(T)):
            nv = last if t == T - 1 else val[t + 1]
            nt = 1.0 - done[t].float()
            delta = r2[t] + nt * gamma * nv - val[t]
            a = delta + nt * gamma * lam * a
            exp_ret[t] = a + val[t]
        assert torch.allclose(ret, exp_ret, rtol=1e-5, atol=1e-5) and torch.allclose(adv, exp_ret - val, rtol=1e-5, atol=1e-5)


def _actor_critic(seed=0):
    torch.manual_seed(seed)
    mk = lambda out: torch.nn.Sequential(torch.nn.Linear(14, 64), torch.nn.ELU(), torch.nn.Linear(64, 64), torch.nn.ELU(), torch.nn.Linear(64, out)).cuda()
    return mk(2), mk(1), torch.tensor([0.7, 1.3], device="cuda")


def test_fused_actor_critic_step_matches_torch_policy_and_plain_step():
    """wl_act_step = rsl_rl ActorCritic.act/evaluate (64x64 ELU MLPs, Gaussian head) + env.step in ONE launch.
    Policy outputs vs a torch fp32 restatement (tolerance: fp32 accumulation order, 2e-5); the env side must be
    BIT-identical to wl_step fed the same sampled actions."""
    _need_gpu()
    import wheeledlab_b200 as wl
    from wheeledlab_b200.policy import act_step, pack_actor_critic
    n = 1531
    actor, critic, std = _actor_critic()
    a = wl.WheeledSim(wl.drift_task(num_envs=n, seed=21), "cuda:0"); b = wl.WheeledSim(wl.drift_task(num_envs=n, seed=21), "cuda:0")
    for s_ in (a, b):
        s_.startup(); s_.reset(None, 0)
    blob = pack_actor_critic(actor, critic, std, 14, "cuda:0")
    obs = a.observe(0, 0)
    dev = "cuda"
    act = torch.empty((n, 2), device=dev); mean = torch.empty((n, 2), device=dev); lp = torch.empty(n, device=dev); val = torch.empty(n, device=dev)
    zs = []
    with torch.no_grad():
        for t in range(40):
            out = tuple(torch.empty_like(x) for x in (obs, lp, torch.empty(n, dtype=torch.uint8, device=dev), torch.empty(n, dtype=torch.uint8, device=dev)))
            act_step(b, obs, blob, act, mean, lp, val, out, None, t)
            m_ref, v_ref = actor(obs), critic(obs).squeeze(-1)
            assert torch.allclose(mean, m_ref, rtol=2e-5, atol=2e-5), (t, (mean - m_ref).abs().max())
            assert torch.allclose(val, v_ref, rtol=2e-5, atol=2e-5), (t, (val - v_ref).abs().max())
            lp_ref = torch.distributions.Normal(mean, std).log_prob(act).sum(-1)
            assert torch.allclose(lp, lp_ref, rtol=1e-4, atol=1e-4), (t, (lp - lp_ref).abs().max())
            zs.append(((act - mean) / std).flatten())
            ref = a.step(act.clone(), t)
            for x, y in zip(out, ref):
                assert torch.equal(x, y), t
            obs = ref[0]
    assert torch.equal(a.groups, b.groups)
    z = torch.cat(zs)
    assert abs(z.mean().item()) < 0.02 and abs(z.var().item() - 1.0) < 0.03          # N(0,1) samples, 122k draws


def test_fused_policy_rollout_graph_equals_eager_act_steps():
    _need_gpu()
    import wheeledlab_b200 as wl
    from wheeledlab_b200.policy import FusedPolicyRollout, act_step, pack_actor_critic
    n, T = 777, 32
    actor, critic, std = _actor_critic(3)
    a = wl.WheeledSim(wl.drift_task(num_envs=n, seed=5), "cuda:0"); b = wl.WheeledSim(wl.drift_task(num_envs=n, seed=5), "cuda:0")
    for s_ in (a, b):
        s_.startup(); s_.reset(None, 0)
    blob = pack_actor_critic(actor, critic, std, 14, "cuda:0")
    roll = FusedPolicyRollout(b, blob, T).capture(0)
    dev = "cuda"
    obs = a.observe(0, 0)
    act = torch.empty((n, 2), device=dev); mean = torch.empty((n, 2), device=dev); lp = torch.empty(n, device=dev); val = torch.empty(n, device=dev)
    for it in range(3):
        slab = roll.run(); torch.cuda.synchronize()
        for k in range(T):
            out = (torch.empty((n, 14), device=dev), torch.empty(n, device=dev), torch.empty(n, dtype=torch.uint8, device=dev), torch.empty(n, dtype=torch.uint8, device=dev))
            act_step(a, obs, blob, act, mean, lp, val, out, None, it * T + k)
            assert torch.equal(slab.actions[k], act) and torch.equal(roll.pol.values[k], val) and torch.equal(roll.pol.log_prob[k], lp), (it, k)
            assert torch.equal(slab.obs[k], out[0]) and torch.equal(slab.rewards[k], out[1])
            obs = out[0]
    assert torch.equal(a.groups, b.groups)
    # storage alignment (rsl_rl RolloutStorage): obs_in[k] is the observation actions[k] / mean[k] / log_prob[k] / values[k]
    # were computed from -- recompute them with torch from the slab alone
    with torch.no_grad():
        for k in (0, 1, T - 1):
            mu = actor(slab.obs_in[k]); v = critic(slab.obs_in[k]).squeeze(-1)
            assert torch.allclose(mu, roll.pol.mean[k], atol=3e-5) and torch.allclose(v, roll.pol.values[k], atol=3e-5), k
            lp_ref = (-0.5 * (((slab.actions[k] - mu) / std.cuda()) ** 2).sum(-1) - torch.log(std.cuda()).sum() - 1.8378770664093453)
            assert torch.allclose(lp_ref, roll.pol.log_prob[k], atol=2e-3), k
            if k + 1 < T:
                assert torch.equal(slab.obs[k], slab.obs_in[k + 1])
    with pytest.raises(wl.WlError):                      # 689-wide elevation observations are not supported by the fused policy
        e = wl.WheeledSim(wl.elevation_task(num_envs=8, seed=1, terrain="procedural"), "cuda:0")
        act_step(e, torch.zeros((8, 689), device=dev), blob, act, mean, lp, val, out, None, 0)


@pytest.mark.parametrize("task", ["drift", "elevation", "visual"])
def test_staged_step_equals_fused_step(task):
    """wl_step_stage_a + wl_step_stage_b (the cut for host-side Python terms) == wl_step, bit for bit, incl. resets,
    episode log, curriculum and the device counter."""
    _need_gpu()
    import wheeledlab_b200 as wl
    n = 333
    mk = {"drift": lambda: wl.drift_task(num_envs=n, seed=17), "elevation": lambda: wl.elevation_task(num_envs=n, seed=17),
          "visual": lambda: wl.visual_task(num_envs=n, seed=17)}[task]
    a, b = wl.WheeledSim(mk(), "cuda:0"), wl.WheeledSim(mk(), "cuda:0")
    for s_ in (a, b):
        s_.startup(); s_.reset(None, 0)
    a.set_kernel_variant(1)                                # same thread-per-env code path as the staged kernels (variants are bit-identical anyway)
    la, lb = torch.zeros(16, device="cuda"), torch.zeros(16, device="cuda")
    steps = 520 if task == "drift" else 230                # crosses episode ends (250 / 200 steps) -> time-out resets + curriculum
    for t in range(steps):
        act = a.synth_actions(t)
        obs, rew, term, trunc = a.step(act, t, log=la); a.flush_log()
        rew_b, bits = b.step_stage_a(act, t)
        obs_b, term_b, trunc_b = b.step_stage_b(bits, t, log=lb); b.flush_log()
        assert torch.equal(rew, rew_b) and torch.equal(obs, obs_b), (task, t)
        assert torch.equal(term, term_b) and torch.equal(trunc, trunc_b), (task, t)
        assert torch.allclose(la, lb, rtol=1e-4, atol=1e-6), (task, t)    # float atomics across warps: order is not fixed
    assert torch.equal(a.groups, b.groups) and torch.equal(a.rew_weight, b.rew_weight)


def test_python_terms_run_between_rewards_and_reset():
    """env.add_reward_term / add_termination_term / add_observation_term: IsaacLab term semantics on the staged step."""
    _need_gpu()
    import wheeledlab_b200 as wl
    n = 257
    plain = wl.ManagerBasedRLEnv(wl.drift_task(num_envs=n, seed=23), device="cuda:0")
    env = wl.ManagerBasedRLEnv(wl.drift_task(num_envs=n, seed=23), device="cuda:0")
    seen = []

    def forward_speed(e, scale=1.0):
        v = e.scene["robot"].data.root_lin_vel_b[:, 0] * scale
        seen.append(v.clone())
        return v

    env.add_reward_term("forward_speed", forward_speed, weight=2.0, params={"scale": 0.5})
    env.add_observation_term("speed_obs", lambda e: e.scene["robot"].data.root_lin_vel_w)
    o0, _ = env.reset(); p0, _ = plain.reset()
    assert o0["policy"].shape == (n, 17) and torch.equal(o0["policy"][:, :14], p0["policy"])
    g = torch.Generator(device="cuda").manual_seed(0)
    sums, n_done = torch.zeros(n, device="cuda"), 0
    for t in range(300):                                   # crosses the 250-step time-out: episode log of the Python term
        act = torch.rand((n, 2), device="cuda", generator=g) * 2 - 1
        o, r, te, tr, ex = env.step(act)
        po, pr, pte, ptr, pex = plain.step(act)
        assert torch.equal(o["policy"][:, :14], po["policy"]) and torch.equal(te, pte) and torch.equal(tr, ptr)
        assert torch.equal(r, pr + seen[-1] * (2.0 * env.step_dt)), t           # built-in total + func * weight * dt
        assert torch.equal(o["policy"][:, 14:], env.scene["robot"].data.root_lin_vel_w)
        for k in pex["log"]:
            assert torch.allclose(ex["log"][k], pex["log"][k], rtol=1e-4, atol=1e-6), (t, k)    # float atomics: summation order
        sums += seen[-1] * (2.0 * env.step_dt)
        done = te | tr
        expect = (sums * done).sum() / done.sum().clamp(min=1) / env.max_episode_length_s       # RewardManager.reset logging
        assert torch.allclose(ex["log"]["Episode_Reward/forward_speed"], expect, rtol=1e-5, atol=1e-7), t
        sums[done] = 0.0
        n_done += int(done.sum())
    assert n_done >= n                                     # every env finished at least one episode (250-step time-out)
    # a Python termination term resets the env in the same step, before the observation is taken
    env3 = wl.ManagerBasedRLEnv(wl.drift_task(num_envs=n, seed=23), device="cuda:0")
    env3.add_termination_term("short_episode", lambda e: e.episode_length_buf >= 7)
    env3.reset()
    for t in range(7):
        pre = env3.episode_length_buf.clone()
        o, r, te, tr, ex = env3.step(torch.zeros((n, 2), device="cuda"))
    fire = pre + 1 >= 7                                    # (an env a built-in term reset earlier is younger)
    assert int(fire.sum()) >= n - 8 and bool(te[fire].all()) and not bool(tr.any())
    assert bool((env3.episode_length_buf[fire] == 0).all())
    assert int(ex["log"]["Episode_Termination/short_episode"]) == int(fire.sum())
    with pytest.raises(NotImplementedError):
        env3.step_host(torch.zeros((n, 2)).pin_memory())


@pytest.mark.parametrize("mode", ["aug", "raw"])
def test_visual_camera_observation_bit_exact(mode):
    """Visual task WITH the camera term (obs = 3200 camera floats + 8 proprio = 3208, PolicyCfg order): the CUDA camera
    kernel (render -> ColorJitter -> 5x5 Gaussian blur -> Grayscale -> Normalize) == the oracle bit for bit, for drawn
    and for explicit augmentation parameters, through wl_step / wl_observe / the staged step, over resets."""
    _need_gpu()
    import wheeledlab_b200 as wl
    n, steps = 96, 60
    spec = wl.visual_task(num_envs=n, seed=7, camera=mode)
    sim = wl.WheeledSim(spec, "cuda:0"); sim.startup(); sim.reset(None, 0)
    orc = O.Oracle(spec.cfg, heightfield=spec.heightfield); orc.startup(); orc.reset(None, 0)
    assert sim.obs_dim == 3208 and orc.obs_dim == 3208
    assert np.array_equal(_bits(sim.observe(0, 2).cpu().numpy()), _bits(orc.observe(0, 2)))
    seen_white = 0.0
    for t in range(steps):
        act = sim.synth_actions(t)
        if t % 3 == 2:                                   # the staged step launches the camera too
            rew, bits = sim.step_stage_a(act, t)
            obs, term, trunc = sim.step_stage_b(bits, t)
        else:
            sim.set_kernel_variant(1 if t % 2 else 4)
            obs, rew, term, trunc = sim.step(act, t)
        o_obs, o_rew, o_term, o_trunc = orc.step(act.cpu().numpy(), t)
        assert np.array_equal(term.cpu().numpy(), o_term) and np.array_equal(trunc.cpu().numpy(), o_trunc), t
        assert np.array_equal(_bits(rew.cpu().numpy()), _bits(o_rew)), t
        got = obs.cpu().numpy()
        assert np.array_equal(_bits(got[:, 3200:]), _bits(o_obs[:, 3200:])), t
        assert np.array_equal(_bits(got[:, :3200]), _bits(o_obs[:, :3200])), (t, np.abs(got[:, :3200] - o_obs[:, :3200]).max())
        seen_white += float((got[:, :3200] > 0).mean())
    assert 0.02 < seen_white / steps < 0.9               # the frames are not blank
    if mode == "aug":                                    # explicit parameters (the golden-vector path), every op order
        buf = torch.zeros((n, 3208), device="cuda")
        for k, order in enumerate(([0, 1, 2, 3], [3, 1, 0, 2], [2, 3, 1, 0])):
            aug = np.array([0.4 + 0.5 * k, 0.85 + 0.1 * k, 1.5 - 0.5 * k, 0.1, [0.1, 1.3, 5.0][k]] + order, dtype=np.float32)
            sim.camera(5, buf, torch.from_numpy(aug).cuda())
            exp = orc.camera(5, aug)
            assert np.array_equal(_bits(buf.cpu().numpy()[:, :3200]), _bits(exp[:, :3200])), k
    with pytest.raises(wl.WlError):                      # single-launch rollout cannot host the second kernel
        from wheeledlab_b200.distributed import RolloutSlab
        sim.rollout(4, 100, RolloutSlab(4, n, 3208, 2, "cuda:0"), torch.empty((4, 16), device="cuda"))


def test_edge_sizes_and_error_paths():
    """N = 1 and ragged N through every entry point added late (staged step, fused policy, camera, GAE, fused rollout),
    empty reset list, and the loud failures of the C-ABI (null / misaligned pointers, wrong task)."""
    _need_gpu()
    import ctypes as C
    import wheeledlab_b200 as wl
    from wheeledlab_b200.distributed import RolloutSlab
    from wheeledlab_b200.learner import compute_returns
    from wheeledlab_b200.policy import act_step, pack_actor_critic
    dev = "cuda"
    actor, critic, std = _actor_critic(1)
    for n in (1, 3, 33):
        a = wl.WheeledSim(wl.drift_task(num_envs=n, seed=2), "cuda:0"); b = wl.WheeledSim(wl.drift_task(num_envs=n, seed=2), "cuda:0")
        orc = O.Oracle(a.spec.cfg); orc.startup(); orc.reset(None, 0)
        for s_ in (a, b):
            s_.startup(); s_.reset(None, 0)
            s_.reset(torch.empty(0, dtype=torch.int64, device=dev), 0)          # empty id list: a no-op
        for t in range(6):
            act = a.synth_actions(t)
            obs, rew, term, trunc = a.step(act, t)
            rew_b, bits = b.step_stage_a(act, t); obs_b, term_b, trunc_b = b.step_stage_b(bits, t)
            o_obs, o_rew, _, _ = orc.step(act.cpu().numpy(), t)
            assert torch.equal(obs, obs_b) and torch.equal(rew, rew_b) and np.array_equal(_bits(obs.cpu().numpy()), _bits(o_obs))
        blob = pack_actor_critic(actor, critic, std, 14, "cuda:0")
        pa = torch.empty((n, 2), device=dev); pm = torch.empty((n, 2), device=dev); lp = torch.empty(n, device=dev); val = torch.empty(n, device=dev)
        out = (torch.empty((n, 14), device=dev), torch.empty(n, device=dev), torch.empty(n, dtype=torch.uint8, device=dev), torch.empty(n, dtype=torch.uint8, device=dev))
        act_step(a, obs, blob, pa, pm, lp, val, out, None, 6)
        ref = b.step(pa.clone(), 6)
        assert all(torch.equal(x, y) for x, y in zip(out, ref)) and torch.allclose(pm, actor(obs), rtol=2e-5, atol=2e-5)
        slab = RolloutSlab(5, n, 14, 2, "cuda:0"); logs = torch.empty((5, 16), device=dev)
        a.rollout(5, 7, slab, logs)
        assert torch.isfinite(slab.obs).all()
        ret, adv = compute_returns(slab.rewards, torch.zeros_like(slab.rewards), torch.zeros(n, device=dev), slab.terminated | slab.truncated, 0.99, 0.95)
        assert torch.isfinite(ret).all() and ret.shape == (5, n)
    cam = wl.WheeledSim(wl.visual_task(num_envs=1, seed=3, camera="aug"), "cuda:0"); cam.startup(); cam.reset(None, 0)
    oc = O.Oracle(cam.spec.cfg, heightfield=cam.spec.heightfield); oc.startup(); oc.reset(None, 0)
    assert np.array_equal(_bits(cam.observe(0).cpu().numpy()), _bits(oc.observe(0)))
    # loud failures
    sim = wl.WheeledSim(wl.drift_task(num_envs=4, seed=1), "cuda:0")
    buf = torch.zeros(64, device=dev)
    assert wl.lib.wl_step(sim._h, None, None, None, None, None, None, 0, None) < 0               # null pointers
    assert wl.lib.wl_step(sim._h, C.c_void_p(buf.data_ptr() + 4), C.c_void_p(buf.data_ptr()), C.c_void_p(buf.data_ptr()), C.c_void_p(buf.data_ptr()),
                          C.c_void_p(buf.data_ptr()), None, 0, None) < 0                      # action not 8-byte aligned
    assert b"aligned" in wl.lib.wl_last_error()
    with pytest.raises(wl.WlError):
        sim.camera(0, torch.zeros((4, 14), device=dev))                                       # no camera term on a drift handle
    with pytest.raises(wl.WlError):
        sim.step_stage_a(sim.synth_actions(0), -1)                                            # the staged step needs the host counter


def test_c_host_example_matches_python_path(tmp_path):
    """examples/c_host/wl_c_host (plain C on the C-ABI: cudaMalloc'd buffers, a config blob, no Python/torch in the process)
    returns bit-for-bit what the Python host gets for the same task: order-independent sums of the output bit patterns."""
    _need_gpu()
    import json
    import shutil
    import subprocess
    import wheeledlab_b200 as wl
    from wheeledlab_b200.dump_config import dump
    root = Path(__file__).resolve().parent.parent
    ex = root / "examples" / "c_host"
    subprocess.run(["make", "-C", str(ex), "CC=" + (shutil.which("gcc", path="/usr/bin") or "gcc")], check=True, stdout=subprocess.DEVNULL)
    n, steps = 1000, 300
    dump("drift", n, str(tmp_path / "cfg.bin"), seed=9)
    r = subprocess.run([str(ex / "wl_c_host"), str(tmp_path / "cfg.bin"), str(steps)], check=True, capture_output=True, text=True, timeout=120)
    got = json.loads(r.stdout.strip().splitlines()[-1])
    sim = wl.WheeledSim(wl.drift_task(num_envs=n, seed=9), "cuda:0"); sim.startup(); sim.reset(None, 0)
    obs_sum = rew_sum = n_term = n_trunc = 0
    for t in range(steps):
        obs, rew, term, trunc = sim.step(sim.synth_actions(t), t)
        obs_sum += int(obs.cpu().numpy().view(np.uint32).astype(np.uint64).sum()); rew_sum += int(rew.cpu().numpy().view(np.uint32).astype(np.uint64).sum())
        n_term += int(term.sum()); n_trunc += int(trunc.sum())
    assert got["envs"] == n and got["steps"] == steps and "sm_90a" in got["build"]
    assert (got["obs_bits_sum"], got["rew_bits_sum"], got["terminated"], got["truncated"]) == (obs_sum, rew_sum, n_term, n_trunc)
    assert n_trunc > 0 and n_term > 0                              # the run crossed the 250-step time-out and saw off-track resets


# ---- oracle parity at BASELINE.json's full sizes and on the action / DR branches (round-2 additions) -------------------
def _oracle_traj(spec, steps, action_fn, threads=8, check_state=True, heightfield=None):
    """CUDA (through the C-ABI) vs the oracle on the same seeded inputs: every output bit-exact every step, the full state at
    the end.  action_fn(sim, t) -> device [N,2] f32.  Returns the number of (env, step) pairs that ended an episode."""
    import wheeledlab_b200 as wl
    sim = wl.WheeledSim(spec, "cuda:0"); sim.startup(); sim.reset(None, 0)
    orc = O.Oracle(spec.cfg, heightfield=spec.heightfield if heightfield is None else heightfield, threads=threads)
    orc.startup(); orc.reset(None, 0)
    n_done = 0
    for t in range(steps):
        act = action_fn(sim, t)
        obs, rew, term, trunc = sim.step(act, t)
        o_obs, o_rew, o_term, o_trunc = orc.step(act.cpu().numpy(), t)
        assert np.array_equal(term.cpu().numpy(), o_term) and np.array_equal(trunc.cpu().numpy(), o_trunc), f"done masks differ at step {t}"
        assert np.array_equal(_bits(rew.cpu().numpy()), _bits(o_rew)), f"reward differs at step {t}"
        assert np.array_equal(_bits(obs.cpu().numpy()), _bits(o_obs)), f"obs differs at step {t}"
        n_done += int((o_term | o_trunc).sum())
    if check_state:
        assert np.array_equal(_bits(_state_groups(sim)), _bits(orc.export_state())), "final state differs"
    return n_done


def _synth(sim, t):
    return sim.synth_actions(t, dist=t % 2)


def _wide_actions(sim, t):
    """N(0, 2): most samples fall outside [-1, 1], so the action term's own bounding (clip / tanh / none) does the work."""
    g = torch.Generator(device="cuda").manual_seed(1000 + t)
    return torch.randn((sim.num_envs, 2), generator=g, device="cuda") * 2.0


def test_drift_4096_envs_bit_exact_vs_oracle():
    """BASELINE configs[1]: RSS_DRIFT_CONFIG at 4096 envs, 60 steps, every output vs the oracle."""
    _need_gpu()
    import wheeledlab_b200 as wl
    assert _oracle_traj(wl.drift_task(num_envs=4096, seed=42), 60, _synth) > 100


def test_elevation_4096_envs_bit_exact_vs_oracle():
    """BASELINE configs[2]: RSS_ELEV_CONFIG at 4096 envs (689-wide observation incl. the 676-ray height scan), 20 steps."""
    _need_gpu()
    import wheeledlab_b200 as wl
    _oracle_traj(wl.elevation_task(num_envs=4096, seed=42), 20, _synth)


def test_hound_4wd_8192_envs_bit_exact_vs_oracle():
    """BASELINE configs[3]: 'HOUND 4WD' = MuSHR with HOUND_SUS_ACTUATOR_CFG (four driven wheels) + Mushr4WDActionCfg + mass /
    friction DR, 8192 envs, 30 steps."""
    _need_gpu()
    import wheeledlab_b200 as wl
    assert _oracle_traj(wl.make_task("hound_4wd", num_envs=8192, seed=42), 30, _synth) > 100


@pytest.mark.parametrize("bounding", [0, 1, 2])        # none / clip / tanh (ackermann_actions.py:123-130)
@pytest.mark.parametrize("kind", [0, 1, 2])            # base Ackermann / RWD / 4WD action terms
def test_action_term_branches_bit_exact_with_out_of_range_actions(kind, bounding):
    """Every (action term, bounding strategy) pair, fed N(0, 2) actions: the in-kernel clip / tanh / linear map is exercised
    against the oracle (round 1's synthetic actions were pre-clipped)."""
    _need_gpu()
    import wheeledlab_b200 as wl
    spec = wl.drift_task(num_envs=512, seed=5, drive="2wd" if kind == 1 else "4wd")
    spec.cfg.action_kind, spec.cfg.bounding = kind, bounding
    if bounding == 0:
        spec.cfg.act_scale[0], spec.cfg.act_scale[1] = 1.0, 0.15        # unbounded actions: keep |delta| away from tan's poles
    _oracle_traj(spec, 120, _wide_actions)


def test_f1tenth_task_bit_exact_vs_oracle():
    """Isaac-F1TenthDriftRL-v0: F1Tenth geometry / masses / actuators (wheeledlab_assets/f1tenth.py, common/actions.py:51-71)."""
    _need_gpu()
    import wheeledlab_b200 as wl
    assert _oracle_traj(wl.make_task("Isaac-F1TenthDriftRL-v0", num_envs=1024, seed=3), 300, _synth) > 100


@pytest.mark.parametrize("variant", [1, 4])
def test_visual_random_dr_variant_bit_exact_vs_oracle(variant):
    """MushrVisualRLRandomEnvCfg (mushr_visual_env_cfg.py:266-299,449-451): abs base mass, abs wheel masses (per-wheel spin
    inertia group WL_G_PIW), 10 friction buckets."""
    _need_gpu()
    import wheeledlab_b200 as wl
    spec = wl.visual_task(num_envs=300, seed=8, randomize=True)
    sim = wl.WheeledSim(spec, "cuda:0"); sim.startup(); sim.reset(None, 0); sim.set_kernel_variant(variant)
    orc = O.Oracle(spec.cfg, heightfield=spec.heightfield); orc.startup(); orc.reset(None, 0)
    assert np.array_equal(_bits(_state_groups(sim)), _bits(orc.export_state()))
    m = sim.groups[9, :, 0]
    assert 3.9 < float(m.min()) and float(m.max()) < 6.9 and float(m.std()) > 0.3
    for t in range(110):
        act = sim.synth_actions(t)
        for x, y in zip(sim.step(act, t), orc.step(act.cpu().numpy(), t)):
            x = x.cpu().numpy()
            assert np.array_equal(_bits(x) if x.dtype == np.float32 else x, _bits(y) if y.dtype == np.float32 else y), t
    assert np.array_equal(_bits(_state_groups(sim)), _bits(orc.export_state()))


def test_vehicle_at_rest_stays_at_rest_on_the_gpu():
    """The implicit DC-motor damper on the CUDA path: zero action, 4WD configuration, the car does not creep (|v| < 1 mm/s)."""
    _need_gpu()
    import wheeledlab_b200 as wl
    spec = wl.visual_task(num_envs=64, seed=3, traversability=np.ones((500, 500), dtype=bool))
    sim = wl.WheeledSim(spec, "cuda:0"); sim.startup(); sim.reset(None, 0)
    sim.groups[2, :, 0:3] = 0; sim.groups[3, :, 0:3] = 0; sim.groups[4] = 0
    zero = torch.zeros((64, 2), device="cuda")
    for t in range(10):
        sim.step(zero, t)
    p0 = sim.root_pos_w.clone()
    for t in range(10, 15):
        sim.step(zero, t)
    assert float((sim.root_pos_w - p0)[:, :2].norm(dim=1).max()) < 1e-3 * 1.0 and float(sim.root_lin_vel_w.abs().max()) < 1e-3
    assert float(sim.wheel_vel.abs().max()) < 1e-2


@pytest.mark.parametrize("mode", ["nccl", "fanout", "mcast", "ce"])
def test_two_process_nccl_gather_equals_single_rank(tmp_path, mode):
    """BASELINE configs[4] at test size: 2 ranks x 2048 envs, the exchanged rollout slab == the slab of one 4096-env process,
    bit for bit (skipped when the box has a single GPU).  mode "nccl": one all_gather_into_tensor of the slab; "fanout": the
    step kernel stores its output rows into the peer's symmetric buffer over NVLink (no collective); "mcast": the same with one
    multimem.st per row, replicated by the NVSwitch (skipped where the fabric has no multicast); "ce": copy-engine pull of the peer's slab
    out of symmetric memory (no SM)."""
    _need_gpu()
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import subprocess, sys
    root = Path(__file__).resolve().parent.parent
    out = tmp_path / "slab.pt"
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", {"nccl": "29731", "fanout": "29733", "ce": "29735", "mcast": "29737"}[mode], str(root / "tools" / "nccl_slab_check.py"), "--out", str(out), "--envs", "2048",
           "--steps", "16", "--mode", mode]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    if mode == "mcast" and "NO_MULTICAST" in r.stdout:
        pytest.skip("no NVSwitch multicast on this box")
    assert r.returncode == 0, r.stderr[-2000:]
    import wheeledlab_b200 as wl
    from wheeledlab_b200.distributed import RolloutSlab
    got = torch.load(out)
    sim = wl.WheeledSim(wl.drift_task(num_envs=4096, seed=42), "cuda:0"); sim.startup(); sim.reset(None, 0)
    slab = RolloutSlab(16, 4096, sim.obs_dim, 2, "cuda:0")
    for t in range(16):
        act = sim.synth_actions(t)
        slab.actions[t].copy_(act)
        sim.step(act, t, out=slab.step_outputs(t))
    torch.cuda.synchronize()
    for name in got:
        assert torch.equal(getattr(slab, name).cpu(), got[name]), name


def test_gym_make_through_the_registry_and_the_reference_smoke_loop():
    """wheeledlab_tasks/__init__.py:14-63 registers `entry_point="isaaclab.envs:ManagerBasedRLEnv"`; with shims/ on the path
    gym.make(id, cfg=...) resolves to the fused-step env.  The loop is the reference's own smoke test
    (wheeledlab_tasks/test/create_and_step_env.py:26-44): reset, then sample-and-step under inference_mode."""
    _need_gpu()
    import sys
    root = Path(__file__).resolve().parent.parent
    sys.path.insert(0, str(root / "shims"))
    import gymnasium as gym
    import wheeledlab_b200 as wl
    for gid in wl.GYM_IDS:                                # the four register() calls of the reference, restated (its package is not on this box)
        gym.register(id=gid, entry_point="isaaclab.envs:ManagerBasedRLEnv", disable_env_checker=True,
                     kwargs={"env_cfg_entry_point": None, "rsl_rl_cfg_entry_point": "x:y"})
    for gid in wl.GYM_IDS:
        spec = wl.make_task(gid, num_envs=48, seed=1)
        assert C.string_at(C.addressof(spec.cfg), 8) == (root / "tests" / "golden" / "cfg_blobs" / f"{gid}.ref.bin").read_bytes()[:8]
        env = gym.make(gid, cfg=spec)
        assert isinstance(env.unwrapped, wl.ManagerBasedRLEnv) and env.num_envs == 48
        import isaaclab.envs
        assert isinstance(env.unwrapped, isaaclab.envs.ManagerBasedRLEnv)
        with torch.inference_mode():
            obs, _ = env.reset()
            for _ in range(12):
                actions = torch.rand((env.num_envs, 2), device="cuda") * 2 - 1
                obs, rew, term, trunc, info = env.step(actions)
            assert obs["policy"].shape == (48, env.spec_obs_dim if hasattr(env, "spec_obs_dim") else spec.obs_dim) and torch.isfinite(obs["policy"]).all()
            assert rew.shape == (48,) and term.dtype == torch.bool and "log" in info
        env.close()


def test_elevation_per_term_termination_masks():
    """TerminationManager.get_term(name) returns the term's OWN mask (ADVICE r1): the union of the non-time-out masks is
    `terminated`, time_out is `truncated`, and each mask's population equals the episode-log count of that term."""
    _need_gpu()
    import wheeledlab_b200 as wl
    env = wl.make("Isaac-MushrElevationRL-v0", num_envs=512, seed=3)
    env.reset()
    names = [n for n, _ in env.spec.termination_names]
    assert names == ["time_out", "cart_out_of_bounds", "stuck", "rollover", "at_goal"]
    seen = {n: 0 for n in names}
    for t in range(230):
        obs, rew, term, trunc, info = env.step(env.sim.synth_actions(t))
        m = {n: env.termination_manager.get_term(n) for n in names}
        assert torch.equal(trunc, m["time_out"])
        assert torch.equal(term, m["cart_out_of_bounds"] | m["stuck"] | m["rollover"] | m["at_goal"])
        if bool((term | trunc).any()):
            for n in names:
                assert int(info["log"]["Episode_Termination/" + n].item()) == int(m[n].sum().item()), (t, n)
        for n in names:
            seen[n] += int(m[n].sum().item())
    assert seen["time_out"] > 0 and seen["stuck"] > 0 and seen["stuck"] != seen["time_out"]
    with pytest.raises(ValueError):
        env.termination_manager.get_term("no_such_term")


def test_fast_div_sqrt_are_ieee():
    """fdiv_norm / fsqrt_norm (the compiler's own MUFU + FFMA fast path, emitted without the range check and slow-path call) give
    the correctly rounded IEEE result over the operand ranges the integrator sub-step feeds them (normal-range operands,
    quotient and intermediates; see wheel_force), and det_atan_ratio<NORM> equals the checked variant."""
    _need_gpu()
    import wheeledlab_b200 as wl
    rng = np.random.default_rng(5)

    def run(op, x, y):
        dx, dy = torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda(); out = torch.empty_like(dx)
        wl._lib.check(wl.lib.wl_test_detmath(op, dx.data_ptr(), dy.data_ptr(), out.data_ptr(), x.size, None))
        torch.cuda.synchronize()
        return out.cpu().numpy()

    n = 4_000_000
    for lo_e, hi_e in ((-40, 14), (-1, 14), (-30, -20)):       # POSITIVE denominators (the sub-step's are), numerators of either sign
        b = (2.0 ** rng.uniform(lo_e, hi_e, n)).astype(np.float32)
        a = (2.0 ** rng.uniform(-40, 14, n)).astype(np.float32) * rng.choice([-1.0, 1.0], n).astype(np.float32)
        a[:1000] = 0.0; a[1000:2000] = 1.0                     # (+0 numerator: the only zero the sub-step can produce)
        assert np.array_equal(_bits(run(9, b, a)), _bits(a / b))
    # mantissa corner cases: all-ones / power-of-two denominators and numerators
    m = np.array([0x3f800000, 0x3fffffff, 0x3f800001, 0x3fc00000, 0x3f7fffff, 0x40490fdb], np.uint32).view(np.float32)
    bb, aa = np.meshgrid(m, m); bb, aa = bb.ravel().copy(), -aa.ravel().copy()
    assert np.array_equal(_bits(run(9, bb, aa)), _bits(aa / bb))
    x = (2.0 ** rng.uniform(-80, 27, n)).astype(np.float32)
    x[:6] = m
    assert np.array_equal(_bits(run(10, x, x)), _bits(np.sqrt(x)))
    den = rng.uniform(0.5, 1.0e3, n).astype(np.float32)
    num = (10.0 * 2.0 ** rng.uniform(-40, 12, n)).astype(np.float32)
    assert np.array_equal(_bits(run(11, den, num)), _bits(run(12, den, num)))


def test_fused_adam_matches_torch_adam_single_rank():
    """wl_dp_adam_step with one rank == torch.optim.Adam (the data-parallel form is covered by the 2-GPU test below)."""
    _need_gpu()
    from wheeledlab_b200.learner import DataParallelAdam
    torch.manual_seed(0)
    mk = lambda: torch.nn.Sequential(torch.nn.Linear(14, 64), torch.nn.ELU(), torch.nn.Linear(64, 64), torch.nn.ELU(), torch.nn.Linear(64, 2)).cuda()
    net, ref = mk(), mk()
    ref.load_state_dict(net.state_dict())
    opt, ropt = DataParallelAdam(net.parameters(), lr=3e-3), torch.optim.Adam(ref.parameters(), lr=3e-3)
    for it in range(20):
        x, y = torch.randn(512, 14, device="cuda"), torch.randn(512, 2, device="cuda")
        opt.zero_grad(); ((net(x) - y) ** 2).mean().backward(); opt.step()
        ropt.zero_grad(); ((ref(x) - y) ** 2).mean().backward(); ropt.step()
    err = max(float((p - q).abs().max()) for p, q in zip(net.parameters(), ref.parameters()))
    assert err < 5e-6, err


def test_two_process_fused_allreduce_adam(tmp_path):
    """DP learner step (SURVEY 8f-2): gradient all-reduce fused into the Adam kernel over symmetric memory, 2 ranks, vs
    torch.optim.Adam on the NCCL-averaged gradient; replicas stay bit-identical (skipped on a single-GPU machine)."""
    _need_gpu()
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import subprocess, sys
    root = Path(__file__).resolve().parent.parent
    out = tmp_path / "ok.txt"
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", "29737", str(root / "tools" / "dp_adam_check.py"), "--out", str(out)]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and out.read_text().startswith("ok"), r.stderr[-2000:]


def test_torch_ops_front_equals_ctypes_host_and_checks_arguments():
    """torch.ops.wheeledlab_b200.{reset, observe_out, step, step_out} drive the same kernels as the ctypes host: two handles of
    the same task stepped side by side (one through each front) stay bit-identical, on a non-default stream and inside a CUDA
    graph; malformed arguments raise RuntimeError naming the argument instead of reaching the kernel."""
    _need_gpu()
    import torch
    import wheeledlab_b200 as wl
    from wheeledlab_b200 import torch_ops
    ops = torch_ops.load()
    n = 1024
    a = wl.WheeledSim(wl.drift_task(num_envs=n, seed=5), "cuda:0"); a.startup(); a.reset(None, 0)
    b = wl.WheeledSim(wl.drift_task(num_envs=n, seed=5), "cuda:0"); b.startup()
    like = torch.empty(1, device="cuda:0")
    ops.reset(b.handle, None, like, 0)
    oa = a.observe(0)
    ob = torch.empty_like(oa); ops.observe_out(b.handle, ob, 0, 0)
    assert torch.equal(oa.view(torch.int32), ob.view(torch.int32))
    s = torch.cuda.Stream()
    for t in range(40):
        act = a.synth_actions(t)
        ra = a.step(act, t)
        if t % 2 == 0:
            rb = ops.step(b.handle, act, t)
        else:                                                    # in-place form, on a side stream
            rb = (torch.empty_like(ra[0]), torch.empty_like(ra[1]), torch.empty_like(ra[2]), torch.empty_like(ra[3]))
            s.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(s):
                ops.step_out(b.handle, act, rb[0], rb[1], rb[2], rb[3], None, t)
            torch.cuda.current_stream().wait_stream(s)
        for x, y in zip(ra, rb):
            assert torch.equal(x.view(torch.uint8), y.view(torch.uint8)), t
    ids = torch.tensor([3, 77, 500], device="cuda:0")
    a.reset(ids, 40); ops.reset(b.handle, ids, like, 40)
    assert torch.equal(a.state_snapshot().view(torch.int32)[: 16 * n * 4], b.state_snapshot().view(torch.int32)[: 16 * n * 4])
    # graph capture through the op
    act = a.synth_actions(41)
    outs = tuple(torch.empty_like(x) for x in ra)
    g = torch.cuda.CUDAGraph(); cs = torch.cuda.Stream(); cs.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(cs), torch.cuda.graph(g, stream=cs):
        ops.step_out(b.handle, act, outs[0], outs[1], outs[2], outs[3], None, 40)
    torch.cuda.current_stream().wait_stream(cs)
    g.replay()
    ra = a.step(act, 40)
    torch.cuda.synchronize()
    for x, y in zip(ra, outs):
        assert torch.equal(x.view(torch.uint8), y.view(torch.uint8))
    # argument checks
    with pytest.raises(RuntimeError, match="action"):
        ops.step(b.handle, torch.zeros(n, 3, device="cuda:0"), 41)
    with pytest.raises(RuntimeError, match="dtype"):
        ops.step(b.handle, torch.zeros(n, 2, device="cuda:0", dtype=torch.float64), 41)
    with pytest.raises(RuntimeError, match="obs"):
        ops.step_out(b.handle, act, torch.empty(n, 13, device="cuda:0"), outs[1], outs[2], outs[3], None, 41)
    with pytest.raises(RuntimeError, match="contiguous"):
        ops.step(b.handle, torch.zeros(2, n, device="cuda:0").t(), 41)
    with pytest.raises(RuntimeError, match="null"):
        ops.step(0, act, 41)
