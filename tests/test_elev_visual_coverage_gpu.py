"""The Elevation and Visual step paths (wl_step_quad_kernel / wl_step_kernel, the height scan, the camera, the blind-Visual
fused rollout) against the CPU oracle across sizes, height-field geometries, scan modes and kernel interleavings.

- Launch geometry: every default dispatch from N = 1 to the first thread-per-env sizes, and the forced thread-per-env
  block sizes; wl_step_launch_info must say which variant and CTA width ran.
- Height-field geometry: rasters of every pitch padding, smaller than the scan window, off the cell lattice at a negative
  origin, at 0.2 m and at the smallest accepted cell, with a raised outside plane, and placed poses on the raster's last
  sample lines -- each in scan modes 0, 1 and 2 and in the quad and thread-per-env variants.
- The scan pipeline's persistent grid around its 792-CTA size on the H100, the lowered reference cfgs, the blind-Visual
  rollout kernel, the camera at ragged sizes, sharded placement, and kernels interleaved on one handle and one stream
  (eagerly, in a CUDA graph and with every step kernel PDL-launched).

Every comparison is bit for bit: obs (proprio and height scan / camera separately), reward and done masks every step, the
full state and the reward weights at the end; the episode-log counts exactly and its sums (float atomics) to rtol 1e-5.
Runs too short to reach an episode end start a third of the envs 3 steps before their time-out.  The file takes about
30 s on one H100 80GB HBM3 (power limit reported as N/A), most of it in the CPU oracle.

The CPU tests at the end restate the scan window's index arithmetic in float32 to show where wl_create must draw the
smallest height-field cell, check that it does, and check that every height-field case changes what the oracle computes."""
import ctypes as C
import math
import os
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent
if __name__ == "__main__":                                  # the WL_PDL=1 child of test_interleaved_kernels_with_pdl_everywhere
    sys.path[:0] = [str(ROOT), str(ROOT / "tests")]

import oracle_lib as O  # noqa: E402

torch = pytest.importorskip("torch")

DEV = "cuda:0"
BLOBS = ROOT / "tests" / "golden" / "cfg_blobs"
QUAD_MAX = 132 * 4 * 32 * 2                                 # WL_QUAD_MAX_ENVS on the H100's 132 SMs
CELL_MIN = 0.0956                                           # the smallest hf_cell wl_create accepts at scan_half 1.25 m (4 digits)


def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


def _launch_info(sim):
    import wheeledlab_b200 as wl
    v, k, s, th = C.c_int32(), C.c_uint32(), C.c_int32(), C.c_int32()
    wl._lib.check(wl.lib.wl_step_launch_info(sim._h, C.byref(v), C.byref(k), C.byref(s), C.byref(th)), "wl_step_launch_info")
    return v.value, th.value


# ---- configs ---------------------------------------------------------------------------------------------------------
def _every_boundary(spec):
    for k in range(spec.cfg.curr_n):
        spec.cfg.curr_every[k] = 1
    return spec


def _elev(n, seed=11, **kw):
    import wheeledlab_b200 as wl
    return _every_boundary(wl.elevation_task(num_envs=n, seed=seed, **kw))


def _vis(n, seed=11, **kw):
    import wheeledlab_b200 as wl
    return _every_boundary(wl.visual_task(num_envs=n, seed=seed, **kw))


def _terrain(ny, nx, seed):
    """A smooth terrain between z = 0.2 and 0.7 with 2 cm of noise: neighbouring samples differ, so a read of the wrong cell
    shows in the scan."""
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:ny, 0:nx].astype(np.float64)
    h = 0.45 + 0.2 * np.sin(0.37 * x + 0.4) * np.cos(0.29 * y - 0.7) + 0.02 * rng.standard_normal((ny, nx))
    return h.astype(np.float32)


# name: (ny, nx, origin, cell, spawn range of x and y, hf_outside_z)
HF_CASES = {
    "nx_mod4_0": (60, 120, (-6.0, -3.0), 0.1, (-6.5, 6.5), 0.0),       # pad_pitch adds 0, 3, 2, 1 columns
    "nx_mod4_1": (60, 121, (-6.0, -3.0), 0.1, (-6.5, 6.5), 0.0),
    "nx_mod4_2": (60, 122, (-6.0, -3.0), 0.1, (-6.5, 6.5), 0.0),
    "nx_mod4_3": (60, 123, (-6.0, -3.0), 0.1, (-6.5, 6.5), 0.0),
    "tiny": (11, 17, (-0.8, -0.5), 0.1, (-19.0, 19.0), 0.0),             # smaller than the window; most windows miss it wholly
    "tiny_centred": (11, 17, (-0.8, -0.5), 0.1, (-1.5, 1.5), 0.0),       # every window holds the whole raster and more
    "off_lattice": (70, 90, (-3.37, 1.13), 0.1, (-3.0, 7.0), 0.0),       # negative window origins: ox & ~3 below zero
    "cell_0.2": (150, 150, (-15.0, -15.0), 0.2, (-19.0, 19.0), 0.0),
    "cell_min": (160, 160, (-7.6, -7.6), CELL_MIN, (-8.0, 8.0), 0.0),
    "outside_z": (61, 61, (-3.0, -3.0), 0.1, (-4.0, 4.0), 0.3),          # wheels cross onto the raised outside plane
}


def _raster_spec(n, seed, ny, nx, origin, cell, alt):
    """Elevation on a _terrain raster.  The pad columns pad_pitch adds hold 5 m instead of a copy of the last column, so a
    read past column nx - 1 shows.  alt (the CPU liveness checks): "shipped" = the shipped raster instead; "edge" = the last
    sample row and column raised by 0.5 m."""
    if alt == "shipped":
        return _elev(n, seed)
    spec = _elev(n, seed, heightfield=_terrain(ny, nx, seed), hf_origin=origin, hf_cell=cell)
    spec.heightfield[:, nx:] = 5.0
    if alt == "edge":
        spec.heightfield[:, nx - 1] += 0.5
        spec.heightfield[ny - 1, :nx] += 0.5
    return spec


def _hf_spec(case, n, seed=5, alt=None):
    """alt: as _raster_spec, or "plane0" = the outside plane at z = 0."""
    ny, nx, origin, cell, spawn, outside_z = HF_CASES[case]
    spec = _raster_spec(n, seed, ny, nx, origin, cell, alt)
    spec.cfg.elev_reset_xy[0], spec.cfg.elev_reset_xy[1] = spawn
    spec.cfg.hf_outside_z = 0.0 if alt == "plane0" else outside_z
    return spec


# placed poses on a 41 x 33 raster at 0.25 m from (0, 0): at yaw 0 every quantity below is exact in binary, so the last ray
# of a base at x = 8.75 lands on fx == nx - 1 (the ix clamp) and at y = 6.75 on fy == ny - 1
PLACED_RASTER = (33, 41, (0.0, 0.0), 0.25)
_up, _dn = (lambda v: float(np.nextafter(np.float32(v), np.float32(np.inf)))), (lambda v: float(np.nextafter(np.float32(v), np.float32(-np.inf))))
PLACED_XY = [(8.75, 4.0), (8.75, 6.75), (1.25, 1.25), (_up(8.75), _up(6.75)), (_dn(8.75), 4.0), (0.0, 0.0), (10.0, 8.0), (_up(10.0), 3.0)]
PLACED_YAW = [0.0, math.pi / 4, -math.pi / 4, math.pi / 2, math.pi]
PLACED_ROLL = [0.0, math.radians(30.0)]                     # tilted: base_link_z moves the ray origin off the root


def _placed_spec(seed=5, alt=None):
    n = len(PLACED_XY) * len(PLACED_YAW) * len(PLACED_ROLL)
    return _raster_spec(n, seed, *PLACED_RASTER, alt)


def _placed_state(state):
    """The state with every env's root put at one of the placed poses, 1 m up."""
    st = state.copy()
    k = 0
    for x, y in PLACED_XY:
        for yaw in PLACED_YAW:
            for roll in PLACED_ROLL:
                cz, sz, cx, sx = math.cos(yaw / 2), math.sin(yaw / 2), math.cos(roll / 2), math.sin(roll / 2)
                st[0, k, :3] = (x, y, 1.0)
                st[1, k] = (cz * cx, cz * sx, sz * sx, sz * cx)          # q_z(yaw) * q_x(roll), (w, x, y, z)
                k += 1
    return st


# ---- the oracle side and the checks ----------------------------------------------------------------------------------
def _pair(spec):
    import wheeledlab_b200 as wl
    sim = wl.WheeledSim(spec, DEV); sim.startup(); sim.reset(None, 0)
    orc = O.Oracle(spec.cfg, heightfield=spec.heightfield, threads=8); orc.startup(); orc.reset(None, 0)
    return sim, orc


def _set_state(sim, orc, st):
    orc.import_state(st)
    sim.groups.copy_(torch.from_numpy(st))
    assert np.array_equal(_bits(sim.groups.cpu().numpy()), _bits(orc.export_state()))


def _near_timeout(sim, orc):
    """Every third env 3 steps before its time-out, on both sides (episode_length_buf is the int32 lane 3 of group 0)."""
    st = orc.export_state()
    ep = st[0, :, 3].view(np.int32).copy()
    ep[::3] = int(sim.cfg.max_episode_length) - 3
    st[0, :, 3] = ep.view(np.float32)
    _set_state(sim, orc, st)


def _split(spec):
    """Column where the proprio part of an obs row starts / ends: (obs[:, :k], obs[:, k:]) = Elevation (proprio, scan),
    Visual with camera (camera, proprio)."""
    if int(spec.cfg.task) == 1:
        return 13, ("proprio", "height scan")
    if int(spec.cfg.vis_cam):
        return int(spec.cfg.vis_cam_w) * (int(spec.cfg.vis_cam_h) - int(spec.cfg.vis_cam_row0)), ("camera", "proprio")
    return 0, ("", "proprio")


def _check_obs(spec, got, ref, what):
    k, names = _split(spec)
    for name, a, b in ((names[0], got[:, :k], ref[:, :k]), (names[1], got[:, k:], ref[:, k:])):
        bad = np.flatnonzero((_bits(a) != _bits(b)).any(axis=1))
        assert bad.size == 0, f"{what}: {name} obs differs at envs {bad[:8]} (max |diff| {np.abs(a - b).max():.3g})"


def _check_step(spec, got, ref, what):
    obs, rew, term, trunc = (x.cpu().numpy() if torch.is_tensor(x) else x for x in got)
    o_obs, o_rew, o_term, o_trunc = ref
    assert np.array_equal(term, o_term) and np.array_equal(trunc, o_trunc), f"{what}: done masks differ"
    assert np.array_equal(_bits(rew), _bits(o_rew)), f"{what}: reward differs"
    _check_obs(spec, obs, o_obs, what)
    return int((o_term | o_trunc).sum())


def _check_log(spec, got, lg, what):
    got = got.cpu().numpy() if torch.is_tensor(got) else got
    m = 9 + len(spec.termination_names)                      # [8] resets, [9 + j] per-term counts
    assert np.allclose(got[:8], lg[:8], rtol=1e-5, atol=0.0), f"{what}: episode-log sums differ"       # float atomics
    assert np.array_equal(got[8:m], lg[8:m].astype(np.float32)), f"{what}: episode-log counts differ"


def _check_end(sim, orc, what=""):
    assert np.array_equal(_bits(sim.groups.cpu().numpy()), _bits(orc.export_state())), f"{what}: final state differs"
    assert np.array_equal(_bits(sim.rew_weight.cpu().numpy()), _bits(orc.weights())), f"{what}: reward weights differ"


def _check_resets(spec, n_done, what=""):
    if spec.cfg.term_enable:
        assert n_done > 0, f"{what}: no env reset in the run"
    else:                                                     # (the lowered play cfgs have no termination term at all)
        assert n_done == 0, f"{what}: an env reset with every termination term off"


def _traj(spec, sim, orc, steps, t0=0, before_step=None, what=""):
    """`steps` wl_steps from t0 with synth_actions, every output every step.  before_step(t) runs on the host first."""
    n_done = 0
    for t in range(t0, t0 + steps):
        if before_step is not None:
            before_step(t)
        act = sim.synth_actions(t, dist=t % 2)
        log = torch.empty(16, device=DEV)
        out = sim.step(act, t, log=log)
        sim.flush_log()                                       # the row of step t is published by the next launch on the handle
        n_done += _check_step(spec, out, orc.step(act.cpu().numpy(), t), f"{what} step {t}")
        _check_log(spec, log, orc.log(), f"{what} step {t}")
    return n_done


def _run(spec, steps, variant=0):
    """`steps` from reset; a run that ends before the first time-out starts from near-time-out episodes."""
    sim, orc = _pair(spec)
    if variant:
        sim.set_kernel_variant(variant)
    w0 = sim.rew_weight.cpu().numpy().copy()
    if steps < spec.cfg.max_episode_length:
        _near_timeout(sim, orc)
    what = f"{spec.name} n={spec.cfg.num_envs}"
    n_done = _traj(spec, sim, orc, steps, what=what)
    _check_end(sim, orc, what)
    _check_resets(spec, n_done, what)
    # the curriculum is applied with the resets at the boundary step: a few envs rarely reset there
    if spec.cfg.curr_n > 0 and spec.cfg.term_enable and steps > spec.cfg.max_episode_length and spec.cfg.num_envs >= 64:
        assert not np.array_equal(sim.rew_weight.cpu().numpy(), w0), f"{what}: the curriculum boundary did not move the weights"
    return sim, orc


# ---- 1. launch geometry ----------------------------------------------------------------------------------------------
GEOMETRY = [                                                  # (N, forced variant, variant, threads per CTA)
    (1, 0, 4, 32), (7, 0, 4, 32), (8, 0, 4, 32), (9, 0, 4, 32), (33, 0, 4, 32), (4095, 0, 4, 32),
    (QUAD_MAX, 0, 4, 32),                                     # the last quad-kernel size
    (QUAD_MAX + 1, 0, 1, 64),                                 # the first thread-per-env size: pick_block's 64-thread CTAs
    (333, 1, 1, 32), (132 * 64 * 2, 1, 1, 64),                # forced thread-per-env: 32-thread CTAs, then 64 from 16 896
]
GEOMETRY_CASES = [(task, *g) for task in ("elevation", "visual") for g in GEOMETRY] + [
    ("visual", 132 * 128 * 4, 0, 1, 128),                     # 67 584: pick_block's 128-thread CTAs (the cheap oracle only)
]


@pytest.mark.gpu
@pytest.mark.parametrize("task,n,forced,variant,threads", GEOMETRY_CASES)
def test_launch_geometry_matches_oracle(task, n, forced, variant, threads):
    """Below 64 envs the run is 260 steps (the Elevation and Visual episode ends at 200 and 50, and the curriculum boundary
    at t = 200); larger runs are 8 steps from near-time-out episodes."""
    _need_gpu()
    spec = (_elev if task == "elevation" else _vis)(n, seed=3)
    sim, _ = _run(spec, 260 if n < 64 else 8, variant=forced)
    assert _launch_info(sim) == (variant, threads), (task, n, _launch_info(sim))


# ---- 2. height-field geometry ----------------------------------------------------------------------------------------
def _modes_traj(spec, sim, orc, steps, what):
    """Step t runs scan mode t % 3; then observe() in each mode against the oracle's."""
    n_done = _traj(spec, sim, orc, steps, before_step=lambda t: sim.set_scan_tma(t % 3), what=what)
    ref = orc.observe(steps, 1)
    for mode in (0, 1, 2):
        sim.set_scan_tma(mode)
        _check_obs(spec, sim.observe(steps, 1).cpu().numpy(), ref, f"{what} observe, scan mode {mode}")
    _check_end(sim, orc, what)
    return n_done


@pytest.mark.gpu
@pytest.mark.parametrize("variant", [4, 1])
@pytest.mark.parametrize("case", list(HF_CASES))
def test_heightfield_geometry_matches_oracle(case, variant):
    _need_gpu()
    spec = _hf_spec(case, 64)
    sim, orc = _pair(spec)
    sim.set_kernel_variant(variant)
    _near_timeout(sim, orc)
    n_done = _modes_traj(spec, sim, orc, 24, f"{case} variant {variant}")
    assert n_done > 0


@pytest.mark.gpu
@pytest.mark.parametrize("variant", [4, 1])
def test_placed_poses_on_the_raster_edges_match_oracle(variant):
    """Bases put on the last sample lines (fx == nx - 1, fy == ny - 1), on the corners, one ulp outside and inside, at six
    yaws and tilted 30 deg; observe() before any step, then steps in every scan mode."""
    _need_gpu()
    spec = _placed_spec()
    sim, orc = _pair(spec)
    sim.set_kernel_variant(variant)
    _set_state(sim, orc, _placed_state(orc.export_state()))
    ref = orc.observe(0, 0)
    for mode in (0, 1, 2):
        sim.set_scan_tma(mode)
        _check_obs(spec, sim.observe(0, 0).cpu().numpy(), ref, f"placed poses, scan mode {mode}")
    _modes_traj(spec, sim, orc, 6, f"placed poses variant {variant}")


# ---- 3. the scan pipeline's persistent grid --------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("n", [791, 792, 793, 1585, 4000])
def test_scan_pipeline_grid_matches_oracle(n):
    """wl_scan_pipe_kernel runs min(N, 132 x 6 = 792) persistent CTAs on the H100: one env per CTA below 792, a second env
    (stage 1) for the first CTAs from 793, a third (stage 0 again: the mbarrier phase flips) from 1585."""
    _need_gpu()
    spec = _elev(n, seed=13)
    sim, orc = _pair(spec)
    sim.set_scan_tma(2)
    _traj(spec, sim, orc, 3, what=f"pipeline n={n}")
    ref = orc.observe(3, 0)
    for mode in (2, 0, 1):
        sim.set_scan_tma(mode)
        _check_obs(spec, sim.observe(3, 0).cpu().numpy(), ref, f"pipeline n={n} observe, scan mode {mode}")
    _check_end(sim, orc)


# ---- 4. the lowered reference cfgs -----------------------------------------------------------------------------------
def _ref_spec(name, n):
    import wheeledlab_b200 as wl
    if "Visual" in name:                                      # the registered Visual cfg observes through the camera
        spec = wl.visual_task(num_envs=n, seed=42, traversability=np.load(BLOBS / "visual_ref_map.npz")["map"], camera="aug")
    else:
        spec = wl.elevation_task(num_envs=n, seed=42)
    raw = (BLOBS / f"{name}.bin").read_bytes()
    assert len(raw) == C.sizeof(spec.cfg)
    C.memmove(C.addressof(spec.cfg), raw, len(raw))
    spec.cfg.num_envs = n
    return _every_boundary(spec)


@pytest.mark.gpu
@pytest.mark.parametrize("name,n,steps", [
    ("Isaac-MushrElevationRL-v0.ref", 333, 205), ("Isaac-MushrElevationRL-v0.play.ref", 333, 205),
    ("Isaac-MushrVisualRL-v0.ref", 64, 55), ("Isaac-MushrVisualRL-v0.play.ref", 64, 55),
])
def test_lowered_reference_cfg_matches_oracle(name, n, steps):
    """Past the first episode end (and the Elevation curriculum boundary at t = 200).  The play cfgs have no termination
    term, so no env may reset."""
    _need_gpu()
    spec = _ref_spec(name, n)
    sim, _ = _run(spec, steps)
    if "Visual" in name:
        assert sim.obs_dim == 3208


# ---- 5. the blind-Visual fused rollout -------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("randomize", [False, True])
@pytest.mark.parametrize("n", [1, 333, 4096])
def test_blind_visual_rollout_matches_steps_and_oracle(n, randomize):
    """wl_rollout_quad_kernel<WL_TASK_VISUAL>: 55 steps in one launch across the 50-step episode end (Visual has no
    curriculum term, so nothing splits the window), in-kernel U[-1, 1] actions, against 55 x (synth_actions + wl_step) on a
    second handle and against the oracle."""
    _need_gpu()
    import wheeledlab_b200 as wl
    from wheeledlab_b200.distributed import RolloutSlab
    K = 55
    spec = _vis(n, seed=21, randomize=randomize)
    a, orc = _pair(spec)
    b = wl.WheeledSim(spec, DEV); b.startup(); b.reset(None, 0)
    slab, logs = RolloutSlab(K, n, 8, 2, DEV), torch.zeros((K, 16), device=DEV)
    a.rollout(K, 0, slab, logs)
    n_done = 0
    for t in range(K):
        what = f"rollout n={n} randomize={randomize} step {t}"
        act = b.synth_actions(t)
        log = torch.empty(16, device=DEV)
        out = b.step(act, t, log=log)
        b.flush_log()
        assert torch.equal(slab.actions[t], act), f"{what}: in-kernel actions differ from synth_actions"
        got = (slab.obs[t], slab.rewards[t], slab.terminated[t], slab.truncated[t])
        assert all(torch.equal(x, y) for x, y in zip(got, out)), f"{what}: rollout differs from wl_step"
        n_done += _check_step(spec, got, orc.step(act.cpu().numpy(), t), what)
        lg = orc.log()
        _check_log(spec, logs[t], lg, what)
        _check_log(spec, log, lg, what)
    _check_end(a, orc, "rollout")
    assert torch.equal(a.groups, b.groups) and torch.equal(a.rew_weight, b.rew_weight)
    assert n_done > 0


# ---- 6. the camera ---------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["raw", "aug"])
@pytest.mark.parametrize("n", [1, 7, 33, 1000])
def test_camera_matches_oracle(n, mode):
    """wl_step (quad and thread-per-env), the staged step and wl_observe, across near-time-out resets."""
    _need_gpu()
    spec = _vis(n, seed=7, camera=mode)
    sim, orc = _pair(spec)
    _near_timeout(sim, orc)
    _check_obs(spec, sim.observe(0, 2).cpu().numpy(), orc.observe(0, 2), "observe before the first step")
    n_done = 0
    for t in range(8):
        what = f"camera {mode} n={n} step {t}"
        act = sim.synth_actions(t)
        log = torch.empty(16, device=DEV)
        if t % 3 == 2:
            rew, bits = sim.step_stage_a(act, t)
            obs, term, trunc = sim.step_stage_b(bits, t, log=log)
            out = (obs, rew, term, trunc)
        else:
            sim.set_kernel_variant(1 if t % 3 else 4)
            out = sim.step(act, t, log=log)
        sim.flush_log()
        n_done += _check_step(spec, out, orc.step(act.cpu().numpy(), t), what)
        _check_log(spec, log, orc.log(), what)
        if t == 4:
            _check_obs(spec, sim.observe(t + 1, 1).cpu().numpy(), orc.observe(t + 1, 1), f"{what}: observe")
    _check_end(sim, orc, f"camera {mode} n={n}")
    assert n_done > 0


@pytest.mark.gpu
@pytest.mark.parametrize("path", ["step", "staged", "drift_step"])
def test_flushed_log_row_is_not_written_again(path):
    """flush_log() publishes the log row of the last step; after it the library writes that step's log buffer no more.  It
    used to: the next launch's janitor published the row again through the same pointer, so a log tensor freed after the
    flush had 16 floats written into whatever reused it (with 1-33 envs the caching allocator handed that block to the
    next staged step's reward, which then differed from the oracle's)."""
    _need_gpu()
    import wheeledlab_b200 as wl
    spec = wl.make_task("drift", num_envs=7, seed=7) if path == "drift_step" else _vis(7, seed=7, camera="raw")
    sim = wl.WheeledSim(spec, DEV); sim.startup(); sim.reset(None, 0)
    logs = [torch.empty(16, device=DEV) for _ in range(4)]
    for t in range(4):
        act = sim.synth_actions(t)
        if path == "staged":
            _, bits = sim.step_stage_a(act, t)
            sim.step_stage_b(bits, t, log=logs[t])
        else:
            sim.step(act, t, log=logs[t])
        sim.flush_log()
        logs[t].fill_(-7.0)                                   # after the flush on the stream: a later write by the library shows
    sim.flush_log()
    torch.cuda.synchronize()
    for t in range(4):
        assert bool((logs[t] == -7.0).all()), f"{path}: the log row of step {t} was written after its flush"


# ---- 7. sharded placement --------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("task", ["elevation", "visual_camera"])
def test_shards_equal_one_run(task):
    """Shards of 333 + 667 envs (env_id_offset 0 / 333) give every output of one 1000-env run bit for bit."""
    _need_gpu()
    import wheeledlab_b200 as wl

    def mk(n, off):
        spec = _elev(n, seed=17, env_id_offset=off) if task == "elevation" else _vis(n, seed=17, env_id_offset=off, camera="aug")
        sim = wl.WheeledSim(spec, DEV); sim.startup(); sim.reset(None, 0)
        L = int(spec.cfg.max_episode_length)
        ids = torch.arange(n, device=DEV)
        sim.episode_length_buf[(ids + off) % 3 == 0] = L - 3
        return sim

    whole, lo, hi = mk(1000, 0), mk(333, 0), mk(667, 333)
    n_done = 0
    for t in range(8):
        act = whole.synth_actions(t)
        a = whole.step(act, t)
        b, c = lo.step(act[:333].contiguous(), t), hi.step(act[333:].contiguous(), t)
        for k, name in enumerate(("obs", "reward", "terminated", "truncated")):
            assert torch.equal(a[k], torch.cat([b[k], c[k]])), f"{task} step {t}: sharded {name} differs"
        n_done += int((a[2] | a[3]).sum())
    assert torch.equal(whole.groups, torch.cat([lo.groups, hi.groups], dim=1))
    assert n_done > 0


# ---- 8. kernels interleaved on one handle ----------------------------------------------------------------------------
def _interleave_spec(task):
    return _elev(64, seed=29) if task == "elevation" else _vis(33, seed=29, camera="aug")


def _script(graph, L):
    """[(op, step counter or scan mode)] until the counter passes the episode length L.  The graph form holds the staged
    step too: it takes the host counter, which is right because the graph is replayed once, from counter 0."""
    ops, t = [], 0
    while t <= L:
        ops.append(("step", t)); t += 1
        ops.append(("reset", t)); ops.append(("observe", t))
        ops.append(("staged", t)); t += 1
        ops.append(("act", t)); t += 1
        ops.append(("thread", t)); t += 1
        ops.append(("scan", (t // 4) % 3))
        ops.append(("step", t)); t += 1
    return ops, t


def _reset_ids(n):
    return np.array(sorted({0, 3, n // 2, n - 1}), np.int64)


def _run_interleaved(task, graph):
    """The sequence of _script on one handle and one stream, no host sync until the end.  Returns every output as numpy."""
    import wheeledlab_b200 as wl
    from wheeledlab_b200.policy import policy_act
    from test_policy_wide_gpu import relu_policy
    spec = _interleave_spec(task)
    n = int(spec.cfg.num_envs)
    sim = wl.WheeledSim(spec, DEV); sim.startup(); sim.reset(None, 0)
    D = sim.obs_dim
    ops, t_end = _script(graph, int(spec.cfg.max_episode_length))
    acts = torch.stack([sim.synth_actions(t) for t in range(t_end)])
    blob = relu_policy(D)
    ids = torch.from_numpy(_reset_ids(n)).to(DEV)
    f32 = lambda *s: torch.empty(s, dtype=torch.float32, device=DEV)
    u8 = lambda *s: torch.empty(s, dtype=torch.uint8, device=DEV)
    bufs = []
    for op, t in ops:
        b = {}
        if op in ("step", "staged", "act", "thread"):
            b = {"obs": f32(n, D), "rew": f32(n), "term": u8(n), "trunc": u8(n), "log": torch.zeros(16, device=DEV)}
            b["act"] = acts[t] if op != "act" else f32(n, 2)
        if op == "act":
            b.update(mean=f32(n, 2), lp=f32(n), val=f32(n))
        if op == "staged":
            b.update(bits=u8(n))
        if op == "observe":
            b = {"obs": f32(n, D)}
        bufs.append(b)
    if graph:                                                 # the policy kernel's shared-memory attribute, outside the capture
        w = wl.WheeledSim(_interleave_spec(task), DEV); w.startup(); w.reset(None, 0)
        policy_act(w, w.observe(0), blob, f32(w.num_envs, 2), f32(w.num_envs, 2), f32(w.num_envs), f32(w.num_envs), 0)
    w0 = sim.rew_weight.clone()

    def body():
        obs_in = None                                         # (every act op follows an observe op)
        for (op, t), b in zip(ops, bufs):
            c = wl.WheeledSim.device_counter_plus(t) if graph and op != "scan" else t
            out = (b.get("obs"), b.get("rew"), b.get("term"), b.get("trunc"))
            if op == "step":
                sim.step(b["act"], c, out=out, log=b["log"])
            elif op == "thread":
                sim.set_kernel_variant(1)
                sim.step(b["act"], c, out=out, log=b["log"])
                sim.set_kernel_variant(0)
            elif op == "scan":
                sim.set_scan_tma(t)
            elif op == "reset":
                sim.reset(ids, t)
            elif op == "observe":
                obs_in = sim.observe(t, 1, out=b["obs"])
            elif op == "staged":
                sim.step_stage_a(b["act"], t, rew=b["rew"], term_bits=b["bits"])
                sim.step_stage_b(b["bits"], t, out=(b["obs"], b["term"], b["trunc"]), log=b["log"])
            elif op == "act":
                policy_act(sim, obs_in, blob, b["act"], b["mean"], b["lp"], b["val"], c)
                sim.step(b["act"], c, out=out, log=b["log"])
        if graph:
            sim.advance_counter(t_end)

    sim.set_step_counter(0)
    if graph:
        g, s = torch.cuda.CUDAGraph(), torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            with torch.cuda.graph(g, stream=s):
                body()
        torch.cuda.current_stream().wait_stream(s)
        sim.set_step_counter(0)                               # (capture moved the host mirror only)
        g.replay()
    else:
        body()
    sim.flush_log()
    torch.cuda.synchronize()
    rec = {"state": sim.groups.cpu().numpy(), "weights": sim.rew_weight.cpu().numpy(), "weights0": w0.cpu().numpy()}
    for k, ((op, _), b) in enumerate(zip(ops, bufs)):
        for f in ("act", "obs", "rew", "term", "trunc", "log"):
            if f in b:
                rec[f"{k}_{f}"] = b[f].cpu().numpy()
    return rec


def _replay_on_oracle(task, graph, rec):
    spec = _interleave_spec(task)
    n = int(spec.cfg.num_envs)
    orc = O.Oracle(spec.cfg, heightfield=spec.heightfield, threads=8); orc.startup(); orc.reset(None, 0)
    ops, _ = _script(graph, int(spec.cfg.max_episode_length))
    n_done = 0
    for k, (op, t) in enumerate(ops):
        what = f"{task} {'graph' if graph else 'eager'}: {op} #{k} at t={t}"
        if op == "scan":
            continue
        if op == "reset":
            orc.reset(_reset_ids(n), t)
        elif op == "observe":
            _check_obs(spec, rec[f"{k}_obs"], orc.observe(t, 1), what)
        else:
            got = tuple(rec[f"{k}_{f}"] for f in ("obs", "rew", "term", "trunc"))
            n_done += _check_step(spec, got, orc.step(rec[f"{k}_act"], t), what)
            _check_log(spec, rec[f"{k}_log"], orc.log(), what)
    assert np.array_equal(_bits(rec["state"]), _bits(orc.export_state())), f"{task}: final state differs"
    assert np.array_equal(_bits(rec["weights"]), _bits(orc.weights())), f"{task}: reward weights differ"
    if spec.cfg.curr_n > 0:
        assert not np.array_equal(rec["weights"], rec["weights0"]), "the curriculum boundary did not move the weights"
    assert n_done > 0, "no auto-reset in the sequence"


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["eager", "graph"])
@pytest.mark.parametrize("task", ["elevation", "visual_camera"])
def test_interleaved_kernels_on_one_handle_match_oracle(task, mode):
    """wl_step, wl_reset of fixed ids, wl_observe, the staged step, wl_policy_act + wl_step (its sampled actions go to the
    oracle), a forced thread-per-env step, a scan-mode switch and wl_step again, repeated past the first episode end (and
    the Elevation curriculum boundary) on one stream."""
    _need_gpu()
    _replay_on_oracle(task, mode == "graph", _run_interleaved(task, mode == "graph"))


@pytest.mark.gpu
def test_interleaved_kernels_with_pdl_everywhere(tmp_path):
    """The same sequences with WL_PDL=1 (the quad and thread-per-env step kernels PDL-launched).  The flag is read when the
    library loads: a child process runs the device side and the oracle checks its outputs here."""
    _need_gpu()
    env = dict(os.environ, WL_PDL="1")
    r = subprocess.run([sys.executable, str(Path(__file__).resolve()), str(tmp_path)], env=env, capture_output=True, text=True,
                       timeout=900, cwd=str(ROOT))
    assert r.returncode == 0, r.stderr[-3000:]
    for task in ("elevation", "visual_camera"):
        for graph in (False, True):
            with np.load(tmp_path / f"{task}_{'graph' if graph else 'eager'}.npz") as z:
                _replay_on_oracle(task, graph, {k: z[k] for k in z.files})


# ---- 9. the scan window and the cell-size limit (CPU) ----------------------------------------------------------------
W, H, SIDE = 44, 40, 26                                      # WL_TILE_W, WL_TILE_H, WL_SCAN_SIDE


def _fma(a, b, c):
    """float32 fmaf (the kernels' fm): the float32 product is exact in float64, so one more rounding gives fmaf but for rare
    double-rounding ties (none matter to a floor)."""
    return np.asarray(np.asarray(a, np.float64) * np.asarray(b, np.float64) + np.asarray(c, np.float64)).astype(np.float32)


def _window_misses(cell, n=20000, seed=0, half=1.25, res=0.1, ext=20.5, tile_h=H):
    """scan_pose / scan_rays index arithmetic in float32 over `n` poses on a +-ext raster of `cell`: the share of poses with
    a ray inside the raster whose 2x2 cell leaves the window (the kernel clamps it into the window: a wrong height).  Half
    the poses take random yaws, half yaw 45 deg and its odd multiples, where the footprint is widest."""
    f = np.float32
    rng = np.random.default_rng(seed)
    nx = int(round(2 * ext / cell)) + 1
    x0 = f(-ext)
    inv = f(1.0) / f(cell)
    reach = f(half) * f(1.41421356237) + f(cell)             # (the library is built with -fmad=false: two roundings)
    bx = rng.uniform(-ext - 1, ext + 1, n).astype(f)
    by = rng.uniform(-ext - 1, ext + 1, n).astype(f)
    yaw = np.where(np.arange(n) % 2 == 0, rng.uniform(-np.pi, np.pi, n), np.pi / 4 * rng.choice([-3, -1, 1, 3], n))
    cy, sy = np.cos(yaw).astype(f), np.sin(yaw).astype(f)
    ox = np.floor((bx - reach - x0) * inv).astype(np.int64) & ~3
    oy = np.floor((by - reach - x0) * inv).astype(np.int64)
    r = np.arange(SIDE * SIDE)
    ry, rx = r // SIDE, r % SIDE
    lx, ly = _fma(rx.astype(f), f(res), f(-half)), _fma(ry.astype(f), f(res), f(-half))
    wx = _fma(cy[:, None], lx[None], _fma(-sy[:, None], ly[None], bx[:, None]))
    wy = _fma(sy[:, None], lx[None], _fma(cy[:, None], ly[None], by[:, None]))
    fx, fy = ((wx - x0) * inv).astype(f), ((wy - x0) * inv).astype(f)
    inside = (fx >= 0) & (fy >= 0) & (fx <= nx - 1) & (fy <= nx - 1)
    ix = np.minimum(np.floor(fx).astype(np.int64), nx - 2)
    iy = np.minimum(np.floor(fy).astype(np.int64), nx - 2)
    ux, uy = ix - ox[:, None], iy - oy[:, None]
    bad = inside & ((ux < 0) | (ux > W - 2) | (uy < 0) | (uy > tile_h - 2))
    return float(bad.any(axis=1).mean())


def _create_error(cell, scan_half=1.25, scan_res=0.1):
    """wl_create's verdict on an Elevation cfg with this cell, without a device: the cfg also carries dr_num_buckets = 0,
    which wl_create refuses after the geometry checks and before its device query.  So "dr_num_buckets" in the message
    means the geometry was accepted; the host buffers are never touched."""
    import wheeledlab_b200 as wl
    spec = wl.elevation_task(num_envs=4, seed=1, heightfield=_terrain(40, 40, 1), hf_origin=(-2.0, -2.0), hf_cell=cell)
    spec.cfg.scan_half, spec.cfg.scan_res = scan_half, scan_res
    spec.cfg.dr_num_buckets = 0
    nbytes = int(wl.lib.wl_state_bytes(4))
    state = np.zeros(nbytes + 256, np.uint8)
    hf = np.zeros(spec.heightfield.size + 4, np.float32)
    p_state = (state.ctypes.data + 255) & ~255
    p_hf = (hf.ctypes.data + 15) & ~15
    h = C.c_void_p()
    rc = wl.lib.wl_create(C.byref(spec.cfg), C.c_void_p(p_state), nbytes, C.c_void_p(p_hf), C.byref(h))
    assert rc != 0 and not h.value
    return wl.lib.wl_last_error().decode()


def test_wl_create_refuses_cells_the_scan_window_cannot_cover():
    assert "dr_num_buckets" in _create_error(0.1) and "dr_num_buckets" in _create_error(0.2)
    assert "dr_num_buckets" in _create_error(CELL_MIN)
    for cell in (0.0955, 0.095, 0.09, 0.05):
        msg = _create_error(cell)
        assert "hf_cell" in msg and "scan_half" in msg, (cell, msg)
    assert "hf_cell" in _create_error(0.1, scan_half=1.35)                          # the footprint grows with scan_half
    assert "scan_half" in _create_error(0.1, scan_res=0.11)                          # rays beyond +-scan_half


def test_scan_window_emulation_draws_the_line_wl_create_draws():
    """At the shipped 0.1 m and at the smallest cell wl_create accepts, no ray of any pose leaves the window; at 0.095 m
    (refused) some do, and at 0.09 and 0.05 m most poses have one.  A window 4 rows shorter (36) already fails at 0.1 m:
    about 70 % of these poses then read a wrong cell (half of them sit at 45 deg yaw, the widest footprint)."""
    assert _window_misses(0.1) == 0 and _window_misses(CELL_MIN) == 0 and _window_misses(0.2) == 0
    assert _window_misses(0.095) > 0.01
    assert _window_misses(0.09) > 0.3 and _window_misses(0.05) > 0.9
    assert 0.6 < _window_misses(0.1, tile_h=36) < 0.8


# what each case's distinctive feature is checked against: the outside plane's height, the last sample row and column
# (read only if the windows reach the raster's far edges: pad columns, ix / iy clamps), else the shipped raster
LIVE_ALT = {"outside_z": "plane0", "placed": "edge", **{f"nx_mod4_{k}": "edge" for k in range(4)}}


@pytest.mark.parametrize("case", list(HF_CASES) + ["placed"])
def test_every_heightfield_case_changes_the_oracle(case):
    """Over the horizon section 2 runs, each height-field case gives other scans or another trajectory than the same cfg
    with its distinctive feature changed: the outside plane at 0 instead of 0.3 m (so a wheel does reach the plane
    branch), the raster's last row and column raised (so windows do reach the far edges), or the shipped raster."""
    alt = LIVE_ALT.get(case, "shipped")
    steps = 6 if case == "placed" else 24

    def run(alt):
        spec = _placed_spec(alt=alt) if case == "placed" else _hf_spec(case, 64, alt=alt)
        orc = O.Oracle(spec.cfg, heightfield=spec.heightfield); orc.startup(); orc.reset(None, 0)
        if case == "placed":
            orc.import_state(_placed_state(orc.export_state()))
        trace = [orc.observe(0, 0)]
        for t in range(steps):
            trace += list(orc.step(orc.synth_actions(t, t % 2), t))
        return trace + [orc.export_state()]

    a, b = run(None), run(alt)
    assert any(not np.array_equal(x, y) for x, y in zip(a, b)), f"{case}: changing it ({alt}) changes nothing the oracle computes"


if __name__ == "__main__":
    out = Path(sys.argv[1])
    for task in ("elevation", "visual_camera"):
        for graph in (False, True):
            np.savez(out / f"{task}_{'graph' if graph else 'eager'}.npz", **_run_interleaved(task, graph))
