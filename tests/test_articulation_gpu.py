"""The articulation view on the device: wl_suspension_kernel (wl_derive_suspension) against the fp32 oracle bit for bit and
the fp64 oracle within the per-element bound of tests/test_articulation_cpu.py, and every joint and root field a Python term
reads through env.scene["robot"].data.

- Rollout states of Drift, HOUND-4WD, F1Tenth, blind and camera Visual, Elevation on the shipped raster and on synthetic
  rasters, at N = 1, 33, 127, 128, 129, 4096 and 8192 (the kernel's 128-thread CTA and its ragged last one), after steps
  that include auto-resets.
- Placed states through the state buffer: the closed-form flat-ground cases, and on a height-field hubs on the last sample
  lines and corners, one ulp inside and outside the raster, outside it (hf_outside_z) and on steep cells.
- The views: joint columns by construction against tasks.MUSHR_JOINT_NAMES, root_lin_vel_b / root_ang_vel_b against an fp64
  inverse rotation, write_root_*_to_sim with and without env_ids, prev_action / last_action, and the reference's two
  joint-view terms against the inputs of the oracle's built-in terms.
- suspension_state() on a side stream and inside a captured graph, and the refusals of wl_derive_suspension.

Each fp64 case prints its largest |err| / bound."""
from __future__ import annotations

import ctypes as C
import math

import numpy as np
import pytest

import oracle_lib as O
from test_articulation_cpu import (G_ANGVEL, G_LINVEL, G_POS, G_QUAT, G_STEER, G_WHEEL, U, check_closed_form,
                                   check_fp64, closed_form_states, make_spec, suspension_ref)

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")
DEV = "cuda:0"
NS = [1, 33, 127, 128, 129, 4096, 8192]


def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


def _terrain(ny, nx, seed, amp=0.2):
    """A smooth terrain around z = 0.45 with 2 cm of noise (neighbouring samples differ)."""
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:ny, 0:nx].astype(np.float64)
    h = 0.45 + amp * np.sin(0.37 * x + 0.4) * np.cos(0.29 * y - 0.7) + 0.02 * rng.standard_normal((ny, nx))
    return h.astype(np.float32)


# name: (ny, nx, origin, cell, spawn range of x and y, hf_outside_z)
HF_CASES = {
    "nx_mod4_3": (60, 123, (-6.0, -3.0), 0.1, (-6.5, 6.5), 0.0),
    "tiny": (11, 17, (-0.8, -0.5), 0.1, (-19.0, 19.0), 0.0),
    "off_lattice": (70, 90, (-3.37, 1.13), 0.1, (-3.0, 7.0), 0.0),
    "cell_min": (160, 160, (-7.6, -7.6), 0.0956, (-8.0, 8.0), 0.0),
    "outside_z": (61, 61, (-3.0, -3.0), 0.1, (-4.0, 4.0), 0.3),
}


def _spec(task, n, seed=3):
    import wheeledlab_b200 as wl
    if task == "visual_camera":
        return wl.visual_task(num_envs=n, seed=seed, camera="aug")
    if task.startswith("elevation:"):
        ny, nx, origin, cell, spawn, outside_z = HF_CASES[task.split(":")[1]]
        spec = wl.elevation_task(num_envs=n, seed=seed, heightfield=_terrain(ny, nx, seed), hf_origin=origin, hf_cell=cell)
        spec.heightfield[:, nx:] = 5.0
        spec.cfg.elev_reset_xy[0], spec.cfg.elev_reset_xy[1] = spawn
        spec.cfg.hf_outside_z = outside_z
        return spec
    return make_spec(task, n, seed)


def _hf(spec):
    return spec.heightfield if int(spec.cfg.task) == 1 else None


def _oracles(spec):
    hf = spec.heightfield if int(spec.cfg.task) != 0 else None
    return O.Oracle(spec.cfg, heightfield=hf), O.Oracle(spec.cfg, heightfield=hf, kind="f64")


def _sim(spec):
    import wheeledlab_b200 as wl
    sim = wl.WheeledSim(spec, DEV)
    sim.startup(); sim.reset(None, 0)
    return sim


def _check(spec, sim, o32, o64, what, min_kept=0.5):
    """Kernel against the fp32 oracle bit for bit and the fp64 oracle within the bound, on the sim's current state."""
    pos, vel = (x.cpu().numpy() for x in sim.suspension_state())
    st = sim.groups.cpu().numpy()
    o32.import_state(st); o64.import_state(st)
    r32, r64 = o32.suspension(), o64.suspension()
    for name, got, ref in (("pos", pos, r32[0]), ("vel", vel, r32[1])):
        bad = np.flatnonzero((_bits(got) != _bits(ref)).any(axis=1))
        assert bad.size == 0, f"{what}: {name} differs from the fp32 oracle at envs {bad[:8]}: {got[bad[:2]]} vs {ref[bad[:2]]}"
    ref = suspension_ref(spec.cfg, st, _hf(spec))
    return check_fp64(pos, vel, ref, r64, what, min_kept), ref


# ---- 1. rollout states -----------------------------------------------------------------------------------------------------
ROLLOUT_CASES = ([(t, n) for t in ("drift", "drift_4wd", "f1tenth_drift", "visual", "visual_camera", "elevation") for n in NS]
                 + [(f"elevation:{c}", n) for c in HF_CASES for n in (129, 4096)])


@pytest.mark.parametrize("task,n", ROLLOUT_CASES)
def test_kernel_matches_oracles_on_rollout_states(task, n):
    """Every third env starts 3 steps before its time-out; the states after 0, 4 and 9 synth_actions steps."""
    _need_gpu()
    spec = _spec(task, n)
    sim = _sim(spec)
    o32, o64 = _oracles(spec)
    ep = sim.groups[G_POS, :, 3].view(torch.int32)
    ep[::3] = int(spec.cfg.max_episode_length) - 3
    done, t = 0, 0
    for steps in (0, 4, 5):
        for _ in range(steps):
            _, _, term, trunc = sim.step(sim.synth_actions(t, dist=t % 2), t)
            done += int((term | trunc).sum())
            t += 1
        assert _check(spec, sim, o32, o64, f"{task} n={n} t={t}")[0] <= 1.0
    if spec.cfg.term_enable:
        assert done > 0


# ---- 2. placed states ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("task", ["drift", "f1tenth_drift"])
def test_closed_form_placed_states(task):
    _need_gpu()
    spec = _spec(task, 64)
    sim = _sim(spec)
    o32, o64 = _oracles(spec)
    st = closed_form_states(spec.cfg, sim.groups.cpu().numpy())
    sim.groups.copy_(torch.from_numpy(st))
    _check(spec, sim, o32, o64, f"{task} closed form")
    pos, vel = (x.cpu().numpy() for x in sim.suspension_state())
    check_closed_form(spec.cfg, st, (pos, vel), suspension_ref(spec.cfg, st), f"{task} closed form")


PLACED_RASTER = (33, 41, (0.0, 0.0), 0.25)                  # fx = 4 x, fy = 4 y exactly: x = 10 is the last line fx = nx - 1
_up = lambda v: float(np.nextafter(np.float32(v), np.float32(np.inf)))
_dn = lambda v: float(np.nextafter(np.float32(v), np.float32(-np.inf)))
EPS0 = 2.0 ** -26                                          # the finest step fl(rho + pc) resolves next to 0
EDGE_XY = [(10.0, 4.0), (5.0, 8.0), (10.0, 8.0), (0.0, 0.0), (0.0, 8.0), (10.0, 0.0),     # last lines and corners
           (_dn(10.0), 4.0), (5.0, _dn(8.0)), (_dn(10.0), _dn(8.0)), (EPS0, EPS0),          # one step inside
           (_up(10.0), 4.0), (5.0, _up(8.0)), (_up(10.0), _up(8.0)), (-EPS0, 3.0), (4.0, -EPS0),  # one step outside
           (12.0, 4.0), (-1.0, -1.0), (2.5, 2.5)]                                             # outside; a cell corner
EDGE_VALUES = [10.0, 8.0, 0.0, _dn(10.0), _up(10.0), _up(8.0), EPS0, -EPS0]   # (below 8 the right hubs step 2 ulp)


def _exact_root(target, rho, com):
    """fp32 root coordinate p with fl(rho + fl(p + com)) == target (the kernel's hub coordinate at the identity rotation), or
    the nearest one when no p gives the target exactly."""
    f = np.float32
    p0 = f(float(target) - float(rho) - float(com))
    ps = np.array([p0] + [np.float32(p0 + k * np.spacing(p0)) for k in range(-64, 65)], np.float32)
    hub = (f(rho) + (ps + f(com)).astype(np.float32)).astype(np.float32)
    return float(ps[np.argmin(np.abs(hub.astype(np.float64) - float(target)))])


def _bilinear(spec, x, y):
    c = spec.cfg
    fx, fy = (x - c.hf_x0) / c.hf_cell, (y - c.hf_y0) / c.hf_cell
    if not (0 <= fx <= c.hf_nx - 1 and 0 <= fy <= c.hf_ny - 1):
        return float(c.hf_outside_z)
    ix, iy = min(int(fx), c.hf_nx - 2), min(int(fy), c.hf_ny - 2)
    tx, ty = fx - ix, fy - iy
    h = spec.heightfield
    za = h[iy, ix] + (h[iy, ix + 1] - h[iy, ix]) * tx
    zb = h[iy + 1, ix] + (h[iy + 1, ix + 1] - h[iy + 1, ix]) * tx
    return float(za + (zb - za) * ty)


def test_hubs_on_the_raster_edges_match_oracles():
    """Each env puts one wheel's hub exactly on an edge point at the identity rotation, 3 mm into the ground, with a
    prescribed velocity; the outside plane is raised to 0.3 m so that a hub read on the wrong side of the border shows."""
    _need_gpu()
    import wheeledlab_b200 as wl
    ny, nx, origin, cell = PLACED_RASTER
    n = 4 * len(EDGE_XY)
    spec = wl.elevation_task(num_envs=n, seed=5, heightfield=_terrain(ny, nx, 5), hf_origin=origin, hf_cell=cell)
    spec.heightfield[:, nx:] = 5.0
    spec.cfg.hf_outside_z = 0.3
    sim = _sim(spec)
    o32, o64 = _oracles(spec)
    c = spec.cfg
    f = np.float32
    com = [f(x) for x in c.com]
    rho_x = [f(f(c.hub_x_rear) - com[0])] * 2 + [f(f(c.hub_x_front) - com[0])] * 2
    rho_y = [f(f(c.hub_y) - com[1]), f(-f(c.hub_y) - com[1])] * 2
    rho_z = f(f(c.hub_z) - com[2])
    st = sim.groups.cpu().numpy()
    rng = np.random.default_rng(2)
    for k, (x, y) in enumerate(EDGE_XY):
        for w in range(4):
            i = 4 * k + w
            zt = _bilinear(spec, x, y)
            px, py = _exact_root(x, rho_x[w], com[0]), _exact_root(y, rho_y[w], com[1])
            pz = zt + float(c.wheel_radius) - 0.003 - float(rho_z) - float(com[2])
            st[G_POS, i, :3] = (px, py, pz)
            st[G_QUAT, i] = (1.0, 0.0, 0.0, 0.0)
            st[G_LINVEL, i, :3] = rng.uniform(-1, 1, 3)
            st[G_ANGVEL, i, :3] = rng.uniform(-2, 2, 3)
    sim.groups.copy_(torch.from_numpy(st))
    worst, ref = _check(spec, sim, o32, o64, "raster edges", min_kept=0.2)   # hubs on cell lines are branch edges
    assert worst <= 1.0
    hub_x = np.array([f(rho_x[i % 4] + f(f(st[G_POS, i, 0]) + com[0])) for i in range(n)])
    hub_y = np.array([f(rho_y[i % 4] + f(f(st[G_POS, i, 1]) + com[1])) for i in range(n)])
    target = np.repeat(np.array(EDGE_XY, np.float32), 4, axis=0)
    for col, hub in ((0, hub_x), (1, hub_y)):                  # the edge coordinates are hit exactly
        edge = np.isin(target[:, col], np.array(EDGE_VALUES, np.float32))
        assert edge.sum() >= 32 and np.array_equal(hub[edge], target[edge, col])


def test_steep_cells_and_tilted_chassis_match_oracles():
    """A raster of 35-50 deg slopes (n_z down to 0.64) under chassis rolled and pitched by up to 25 deg."""
    _need_gpu()
    import wheeledlab_b200 as wl
    ny, nx = 48, 56
    y, x = np.mgrid[0:ny, 0:nx].astype(np.float64)
    h = (0.1 * (x % 8) + 0.12 * np.abs((y % 6) - 3) + 0.02 * np.random.default_rng(7).standard_normal((ny, nx))).astype(np.float32)
    n = 4096
    spec = wl.elevation_task(num_envs=n, seed=7, heightfield=h, hf_origin=(-2.0, -2.0), hf_cell=0.1)
    spec.heightfield[:, nx:] = 5.0
    sim = _sim(spec)
    o32, o64 = _oracles(spec)
    rng = np.random.default_rng(3)
    st = sim.groups.cpu().numpy()
    roll, pitch, yaw = (rng.uniform(-a, a, n) for a in (math.radians(25), math.radians(25), math.pi))
    cr, sr, cp, sp, cy, sy = np.cos(roll / 2), np.sin(roll / 2), np.cos(pitch / 2), np.sin(pitch / 2), np.cos(yaw / 2), np.sin(yaw / 2)
    st[G_QUAT] = np.stack([cr * cp * cy + sr * sp * sy, sr * cp * cy - cr * sp * sy, cr * sp * cy + sr * cp * sy,
                           cr * cp * sy - sr * sp * cy], axis=1)
    xy = rng.uniform(-1.9, 3.4, (n, 2))
    st[G_POS, :, :2] = xy
    st[G_POS, :, 2] = [_bilinear(spec, a, b) for a, b in xy]
    st[G_POS, :, 2] += rng.uniform(-0.06, 0.02, n)
    st[G_LINVEL, :, :3] = rng.uniform(-2, 2, (n, 3))
    st[G_ANGVEL, :, :3] = rng.uniform(-3, 3, (n, 3))
    sim.groups.copy_(torch.from_numpy(st))
    worst, ref = _check(spec, sim, o32, o64, "steep cells")
    assert worst <= 1.0
    touching = (ref["comp"].v > 0) & ~ref["branch"]
    assert touching.sum() > n // 2 and ref["n_z"].v[touching].min() < 0.7


# ---- 3. the views -----------------------------------------------------------------------------------------------------------
def _env(task, n, seed=1):
    import wheeledlab_b200 as wl
    env = wl.ManagerBasedRLEnv(_spec(task, n, seed), device=DEV)
    env.reset()
    return env


def test_joint_columns_follow_the_joint_names():
    """Distinct wheel speeds, steer angles and steer rates; env k lowers corner k % 4 (bl, br, fl, fr) deepest and gives it
    the fastest compression.  Every name in MUSHR_JOINT_NAMES must read its own joint."""
    _need_gpu()
    from wheeledlab_b200.tasks import MUSHR_JOINT_NAMES
    n = 8
    env = _env("drift", n)
    sim, robot = env.sim, env.scene["robot"]
    c = sim.cfg
    st = sim.groups.cpu().numpy()
    r, hz = float(np.float32(c.wheel_radius)), float(np.float32(c.hub_z))
    for k in range(n):
        sx, sy = [(-1, 1), (-1, -1), (1, 1), (1, -1)][k % 4]
        a, b = math.radians(1.0) * sx, math.radians(-1.0) * sy                   # pitch lowers the front, roll the right
        qy, qx = (math.cos(a / 2), 0, math.sin(a / 2), 0), (math.cos(b / 2), math.sin(b / 2), 0, 0)
        st[G_QUAT, k] = (qx[0] * qy[0], qx[1] * qy[0], qx[0] * qy[2], qx[1] * qy[2])
        st[G_POS, k, :3] = (0.0, 0.0, r - hz - 0.002)
        st[G_LINVEL, k, :3] = (0.0, 0.0, 0.0)
        st[G_ANGVEL, k, :3] = (0.5 * b / abs(b), 0.5 * a / abs(a), 0.0)            # the same corner moves down fastest
        st[G_WHEEL, k] = (10 + k, 20 + k, 30 + k, 40 + k)
        st[G_STEER, k] = (0.1 + 0.01 * k, -0.2 - 0.01 * k, 1.5 + k, -2.5 - k)
    sim.groups.copy_(torch.from_numpy(st))
    d = robot.data
    jp, jv = d.joint_pos, d.joint_vel
    sp, sv = sim.suspension_state()
    assert torch.equal(jp[:, 0:4], torch.zeros(n, 4, device=DEV))              # wheel angles are not tracked
    want_pos = {"throttle": None, "steer": torch.from_numpy(st[G_STEER, :, 0:2]), "suspension": sp.cpu()}
    want_vel = {"throttle": torch.from_numpy(st[G_WHEEL]), "steer": torch.from_numpy(st[G_STEER, :, 2:4]), "suspension": sv.cpu()}
    order = {"back_left": 0, "back_right": 1, "front_left": 2, "front_right": 3}
    for name in MUSHR_JOINT_NAMES:
        ids, names = robot.find_joints(name)
        assert names == [name] and len(ids) == 1
        kind = name.rsplit("_", 1)[1]
        side = name.rsplit("_wheel_", 1)[0]
        j = order[side] - (2 if kind == "steer" else 0)
        if want_pos[kind] is not None:
            assert torch.equal(jp[:, ids].cpu()[:, 0], want_pos[kind][:, j]), name
        assert torch.equal(jv[:, ids].cpu()[:, 0], want_vel[kind][:, j]), name
        if kind == "suspension":                                                # env k: corner k % 4 deepest and fastest
            mine = torch.arange(n, device=DEV) % 4 == order[side]
            for view in (jp, jv):
                assert (view[mine, ids[0]] == view[mine, 6:10].max(dim=1).values).all(), name
                assert (view[mine, ids[0]] > view[mine, 6:10].min(dim=1).values).all(), name


def _quats(rng, n):
    q = [(1.0, 0.0, 0.0, 0.0), (0.0, 1.0, 0.0, 0.0), (0.0, 0.0, 1.0, 0.0), (0.0, 0.0, 0.0, 1.0),    # identity, 180 about x, y, z
         (1.0, 1e-4, -2e-4, 3e-4), (math.cos(1e-3), 0.0, 0.0, math.sin(1e-3))]                   # near identity
    r = rng.standard_normal((n - len(q), 4))
    r /= np.linalg.norm(r, axis=1, keepdims=True)
    q = np.concatenate([np.array(q), r])
    q[len(q) // 2:] *= (1.0 + rng.uniform(-5e-7, 5e-7, (len(q) - len(q) // 2, 1)))                 # non-unit by a few ulp
    return q.astype(np.float32)


def test_root_velocity_views_match_an_fp64_inverse_rotation():
    """root_*_vel_b = q^-1 v q.  In fp32 the view's v - w t + xyz x t (t = 2 xyz x v) is within u |v| (2 + 24 |q|^2) of the
    same expression in fp64: t's components within 4 u |q| |v|, w t within 6 u |q|^2 |v|, v - w t within u |v| (1 + 8 |q|^2),
    xyz x t within 12 u |q|^2 |v| and the last add within u |v| (1 + 4 |q|^2).  That expression is |q|^2 R(q/|q|)^T v +
    (1 - |q|^2) v, so a non-unit q adds 2 ||q|^2 - 1| |v| against the rotation by q/|q|."""
    _need_gpu()
    n = 4096
    env = _env("drift", n)
    sim, d = env.sim, env.scene["robot"].data
    rng = np.random.default_rng(4)
    q = _quats(rng, n)
    v = (rng.standard_normal((n, 3)) * np.exp(rng.uniform(-8, 3, (n, 1)))).astype(np.float32)
    w = (rng.standard_normal((n, 3)) * np.exp(rng.uniform(-8, 3, (n, 1)))).astype(np.float32)
    sim.groups[G_QUAT] = torch.from_numpy(q).to(DEV)
    sim.groups[G_LINVEL, :, :3] = torch.from_numpy(v).to(DEV)
    sim.groups[G_ANGVEL, :, :3] = torch.from_numpy(w).to(DEV)
    q64 = q.astype(np.float64)
    s2 = (q64 * q64).sum(axis=1)
    qh = q64 / np.sqrt(s2)[:, None]
    a, b, cc, dd = qh.T
    R = np.stack([1 - 2 * (cc * cc + dd * dd), 2 * (b * cc - a * dd), 2 * (b * dd + a * cc),
                  2 * (b * cc + a * dd), 1 - 2 * (b * b + dd * dd), 2 * (cc * dd - a * b),
                  2 * (b * dd - a * cc), 2 * (cc * dd + a * b), 1 - 2 * (b * b + cc * cc)], axis=1).reshape(n, 3, 3)
    worst = 0.0
    for name, got, x in (("root_lin_vel_b", d.root_lin_vel_b, v), ("root_ang_vel_b", d.root_ang_vel_b, w)):
        x64 = x.astype(np.float64)
        ref = np.einsum("nji,nj->ni", R, x64)
        mag = np.linalg.norm(x64, axis=1)
        bound = (U * (2 + 24 * s2) + 2 * np.abs(s2 - 1) + 1e-15) * mag
        err = np.abs(got.cpu().numpy().astype(np.float64) - ref).max(axis=1)
        ratio = err / bound
        assert (ratio <= 1.0).all(), f"{name}: env {ratio.argmax()} |err| {err.max():.3g} > bound {bound[ratio.argmax()]:.3g}"
        worst = max(worst, float(ratio.max()))
    assert np.allclose(d.root_lin_vel_b.cpu().numpy()[1], v[1] * [1, -1, -1], rtol=1e-6, atol=0)   # 180 deg about x
    print(f"root velocity views: largest |err| / bound {worst:.3g}")


@pytest.mark.parametrize("ids", [None, [0, 5, 7, 63]])
def test_write_root_state_changes_only_the_named_envs_and_the_next_step_reads_it(ids):
    _need_gpu()
    n = 64
    env = _env("drift", n)
    sim, robot = env.sim, env.scene["robot"]
    env.step(sim.synth_actions(0))
    before = sim.state_snapshot()
    k = n if ids is None else len(ids)
    rng = np.random.default_rng(5)
    qq = rng.standard_normal((k, 4)); qq /= np.linalg.norm(qq, axis=1, keepdims=True)
    pose = torch.from_numpy(np.concatenate([rng.uniform(-1, 1, (k, 2)), np.full((k, 1), 0.12), qq], axis=1).astype(np.float32)).to(DEV)
    vel = torch.from_numpy(rng.uniform(-1, 1, (k, 6)).astype(np.float32)).to(DEV)
    env_ids = None if ids is None else torch.tensor(ids, device=DEV)
    robot.write_root_pose_to_sim(pose, env_ids=env_ids)
    robot.write_root_velocity_to_sim(vel, env_ids=env_ids)
    sel = np.arange(n) if ids is None else np.array(ids)
    g = sim.groups
    assert torch.equal(g[G_POS, sel, :3], pose[:, :3]) and torch.equal(g[G_QUAT, sel], pose[:, 3:7])
    assert torch.equal(g[G_LINVEL, sel, :3], vel[:, :3]) and torch.equal(g[G_ANGVEL, sel, :3], vel[:, 3:6])
    after = sim.state_snapshot()
    changed = (after.view(torch.int32) != before.view(torch.int32)).cpu().numpy()
    expect = np.zeros_like(changed)
    gv = expect[: 16 * n * 4].reshape(16, n, 4)
    for grp, cols in ((G_POS, slice(0, 3)), (G_QUAT, slice(0, 4)), (G_LINVEL, slice(0, 3)), (G_ANGVEL, slice(0, 3))):
        gv[grp, sel, cols] = True
    assert not (changed & ~expect).any(), "write_root_*_to_sim changed something it was not asked to"
    orc = O.Oracle(sim.cfg)
    orc.import_state(sim.groups.cpu().numpy())
    act = sim.synth_actions(1)
    obs, rew, term, trunc, _ = env.step(act)
    o_obs, o_rew, o_term, o_trunc = orc.step(act.cpu().numpy(), 1)
    assert np.array_equal(_bits(obs["policy"].cpu().numpy()), _bits(o_obs)) and np.array_equal(_bits(rew.cpu().numpy()), _bits(o_rew))
    assert np.array_equal(_bits(sim.groups.cpu().numpy()), _bits(orc.export_state()))


def test_prev_and_last_action_after_two_steps():
    _need_gpu()
    n = 256
    env = _env("drift", n)
    a0 = torch.rand(n, 2, device=DEV) * 2 - 1
    a1 = torch.rand(n, 2, device=DEV) * 2 - 1
    _, _, t0, u0, _ = env.step(a0)
    _, _, t1, u1, _ = env.step(a1)
    kept = ~(t0 | u0 | t1 | u1)                                   # (an auto-reset restarts the action history)
    assert kept.float().mean() > 0.9
    assert torch.equal(env.action_manager.action[kept], a1[kept]) and torch.equal(env.sim.last_action[kept], a1[kept])
    assert torch.equal(env.action_manager.prev_action[kept], a0[kept]) and torch.equal(env.sim.prev_action[kept], a0[kept])


def test_reference_joint_view_terms_read_what_the_builtin_terms_read():
    """forward_wheel_spin / stuck (Elevation) sum the throttle-joint speeds; turn_left_go_right (Drift) means the steer-joint
    positions.  Through the shim's mdp.joint_vel / mdp.joint_pos they must read the omega and steer the oracle's terms take."""
    _need_gpu()
    import sys
    from pathlib import Path
    shims = str(Path(__file__).resolve().parent.parent / "shims")
    if shims not in sys.path:
        sys.path.insert(0, shims)
    from isaaclab.envs import mdp
    for task, steps in (("elevation", 6), ("drift", 6)):
        env = _env(task, 256)
        for t in range(steps):
            env.step(env.sim.synth_actions(t))
        st = env.sim.groups.cpu().numpy()
        robot = env.scene["robot"]
        if task == "elevation":
            ids = robot.find_joints(".*_throttle")[0]
            jv = mdp.joint_vel(env)[..., ids]
            assert np.array_equal(_bits(jv.cpu().numpy()), _bits(st[G_WHEEL]))
            om = st[G_WHEEL].astype(np.float64)
            s = torch.sum(jv, dim=-1).cpu().numpy()
            assert (np.abs(s - om.sum(axis=1)) <= 3 * U * np.abs(om).sum(axis=1)).all()
        else:
            ids = robot.find_joints(".*_steer")[0]
            jp = mdp.joint_pos(env)[..., ids]
            assert np.array_equal(_bits(jp.cpu().numpy()), _bits(st[G_STEER, :, 0:2]))
            mean = jp.mean(dim=-1).cpu().numpy()
            assert np.array_equal(_bits(mean), _bits((st[G_STEER, :, 0] + st[G_STEER, :, 1]) / np.float32(2)))


# ---- 4. streams, graphs and refusals ---------------------------------------------------------------------------------------
def test_side_stream_and_captured_graph_equal_the_eager_call():
    _need_gpu()
    n, K = 4096, 5
    a, b = _sim(_spec("elevation", n, 9)), _sim(_spec("elevation", n, 9))
    acts = [a.synth_actions(t) for t in range(K)]
    for t in range(K):
        b.step(acts[t], t)
    eager = [x.clone() for x in b.suspension_state()]
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        on_side = [x.clone() for x in b.suspension_state()]
    torch.cuda.current_stream().wait_stream(side)
    a.set_step_counter(0)
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        with torch.cuda.graph(g, stream=s):
            for k in range(K):
                a.step(acts[k], a.device_counter_plus(k))
            graphed = a.suspension_state()
            a.advance_counter(K)
    torch.cuda.current_stream().wait_stream(s)
    a.set_step_counter(0)                                      # (capture moved the host mirror only)
    g.replay()
    torch.cuda.synchronize()
    for x, y, z in zip(eager, on_side, graphed):
        assert np.array_equal(_bits(x.cpu().numpy()), _bits(y.cpu().numpy()))
        assert np.array_equal(_bits(x.cpu().numpy()), _bits(z.cpu().numpy()))
    assert np.array_equal(_bits(a.groups.cpu().numpy()), _bits(b.groups.cpu().numpy()))


def test_null_or_misaligned_outputs_are_refused_by_name():
    _need_gpu()
    import wheeledlab_b200 as wl
    sim = _sim(_spec("drift", 64))
    buf = torch.zeros(2 * 64 * 4 + 4, device=DEV)
    p, v = buf.data_ptr(), buf.data_ptr() + 64 * 16
    call = lambda a, b: wl.lib.wl_derive_suspension(sim._h, C.c_void_p(a) if a else None, C.c_void_p(b) if b else None, None)
    for args in ((0, v), (p, 0), (0, 0)):
        assert call(*args) != 0 and b"wl_derive_suspension" in wl.lib.wl_last_error()
    for args in ((p + 4, v), (p, v + 8)):
        assert call(*args) != 0 and b"wl_derive_suspension" in wl.lib.wl_last_error() and b"aligned" in wl.lib.wl_last_error()
    assert wl.lib.wl_derive_suspension(None, C.c_void_p(p), C.c_void_p(v), None) != 0
    assert call(p, v) == 0
    torch.cuda.synchronize()
