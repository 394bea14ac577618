"""The derived suspension joint state (wl_derive_suspension, the oracle's wlo_derive_suspension) without a GPU: closed-form
placed states that pin what the numbers mean, and the fp32 oracle against the fp64 oracle within a per-element rounding
bound on rollout states of every task.  tests/test_articulation_gpu.py runs the kernel against both with the same machinery.

Conventions (DESIGN §3): wheel order [bl, br, fl, fr]; pos = clamp(comp, -susp_travel, +susp_travel), where comp is how far
the undeflected wheel would reach into the ground along the ground normal (positive = compressed, negative = extended, the
wheel hangs clear below -susp_travel); vel = d(comp)/dt while the wheel touches (comp > 0) and exactly 0 when it does not.

``TV`` holds an fp64 value v and a bound e on |fp32 result - v|, where the fp32 result is what the kernel's sequence of fp32
operations gives on the same fp32 inputs.  The sequence is csrc/wl_api.cu ``wl_suspension_kernel`` with the helpers of
wl_device.cuh / wl_step.cuh; the library is built with -fmad=false, so every fmaf is explicit and nothing else fuses:

* each rounding adds (u + u64) (|v| + e) + 2^-149, u = 2^-24: the fp32 rounding, the fp64 reference's own (u64 = 2^-52
  covers its two roundings of a*b + c) and fp32's smallest subnormal near underflow;
* a product or fma propagates |a| e_b + |b| e_a + e_a e_b + e_c (exact); 2x and -x are exact; sqrt and 1/x of s >= 1
  propagate e / (sqrt(s) + sqrt(s - e)) and e / (s (s - e)) (exact, s - e > 0);
* the chains, in the kernel's order: R = rotmat(q) (two fmas and a product per entry), dot3 = fma(a0, b0, fma(a1, b1,
  a2 * b2)) (3 roundings), hub = R rho + (p + R com) (dot3 then 2 adds), height-field sample (d_inv_hf_cell is within its own
  rounding of 1 / cell: that difference is carried exactly), comp = fma(-(hub_z - zt), n_z, r), nb = R^T n, rc = fma(-r,
  nb, rho), vc = cross(wb, rc) + vb, vel = -dot3(nb, vc).  So the bound of pos is built from |rho|, |hub_z|, |zt| and the
  rotation terms, and that of vel from |vb| and |wb| |rc| through the dot product;
* clamp is 1-Lipschitz; the comp > 0 select and the height-field's cell choice and inside test are branches: a wheel whose
  comp lies within its bound of 0 or of +-susp_travel, or whose cell coordinate lies within its bound of a cell line or of
  the raster's border, is left out of the fp64 check (it is still checked against the fp32 oracle, bit for bit).

Every fp64 check prints the largest |err| / bound it saw."""
from __future__ import annotations

import math

import numpy as np
import pytest

import oracle_lib as O

U = 2.0 ** -24                      # fp32 unit roundoff
U64 = 2.0 ** -52                    # the fp64 reference's two roundings of a*b + c
ETA = 2.0 ** -149                   # fp32's smallest subnormal
G_POS, G_QUAT, G_LINVEL, G_ANGVEL, G_WHEEL, G_STEER, G_ACTION = range(7)
G_CMDB = 14
TASKS = ["drift", "drift_4wd", "f1tenth_drift", "visual", "elevation"]


class TV:
    """fp64 value v and a bound e on |fp32 result - v| (numpy arrays of one shape)."""
    __slots__ = ("v", "e")

    def __init__(self, v, e=None):
        self.v = np.asarray(v, np.float64)
        self.e = np.zeros_like(self.v) if e is None else np.asarray(e, np.float64)

    def __neg__(self):
        return TV(-self.v, self.e)

    def __add__(self, o):
        return rnd(self.v + o.v, self.e + o.e)

    def __sub__(self, o):
        return rnd(self.v - o.v, self.e + o.e)

    def __mul__(self, o):
        return rnd(self.v * o.v, _prod_e(self, o))

    def twice(self):
        return TV(2.0 * self.v, 2.0 * self.e)


def _prod_e(a, b):
    return np.abs(a.v) * b.e + np.abs(b.v) * a.e + a.e * b.e


def rnd(v, e):
    return TV(v, e + (U + U64) * (np.abs(v) + e) + ETA)


def fm(a, b, c):
    return rnd(a.v * b.v + c.v, _prod_e(a, b) + c.e)


def const(x, shape=()):
    return TV(np.full(shape, float(np.float32(x))))


def tv_sqrt(s):
    v = np.sqrt(s.v)
    return rnd(v, s.e / (v + np.sqrt(np.maximum(s.v - s.e, 0.0))))


def tv_recip(s):
    assert (s.v - s.e > 0).all()
    return rnd(1.0 / s.v, s.e / (s.v * (s.v - s.e)))


def dot3(a, b):
    return fm(a[0], b[0], fm(a[1], b[1], a[2] * b[2]))


def rotmat(w, x, y, z):
    one, m2 = const(1.0, w.v.shape), const(-2.0, w.v.shape)
    return [fm(m2, fm(y, y, z * z), one), fm(x, y, -(w * z)).twice(), fm(x, z, w * y).twice(),
            fm(x, y, w * z).twice(), fm(m2, fm(x, x, z * z), one), fm(y, z, -(w * x)).twice(),
            fm(x, z, -(w * y)).twice(), fm(y, z, w * x).twice(), fm(m2, fm(x, x, y * y), one)]


def rot(R, a):
    return [dot3(R[0:3], a), dot3(R[3:6], a), dot3(R[6:9], a)]


def rotT(R, a):
    return [dot3([R[0], R[3], R[6]], a), dot3([R[1], R[4], R[7]], a), dot3([R[2], R[5], R[8]], a)]


def cross(a, b):
    return [fm(a[1], b[2], -(a[2] * b[1])), fm(a[2], b[0], -(a[0] * b[2])), fm(a[0], b[1], -(a[1] * b[0]))]


def _bcast(t, shape):
    return TV(np.broadcast_to(t.v, shape), np.broadcast_to(t.e, shape))


def _terrain(cfg, hf, x, y):
    """Height z, normal n and a flag of wheels whose cell choice or inside test the rounding could flip (hf_sample +
    heightfield_at)."""
    shape = x.v.shape
    up = [TV(np.zeros(shape)), TV(np.zeros(shape)), TV(np.ones(shape))]
    if int(cfg.task) != 1 or hf is None:
        return TV(np.zeros(shape)), up, np.zeros(shape, bool)
    nx, ny, pitch = int(cfg.hf_nx), int(cfg.hf_ny), int(cfg.hf_pitch)
    inv64 = 1.0 / float(np.float32(cfg.hf_cell))
    inv = TV(np.full(shape, inv64), np.full(shape, abs(float(np.float32(inv64)) - inv64)))   # d_inv_hf_cell vs 1 / cell
    fx = (x - const(cfg.hf_x0, shape)) * inv
    fy = (y - const(cfg.hf_y0, shape)) * inv
    inside = (fx.v >= 0) & (fy.v >= 0) & (fx.v <= nx - 1) & (fy.v <= ny - 1)
    edge = np.zeros(shape, bool)
    for f, m in ((fx, nx), (fy, ny)):
        lo, hi = f.v - f.e, f.v + f.e
        edge |= (lo < 0) & (hi >= 0) | (lo <= m - 1) & (hi > m - 1)                       # the inside test
        cell_line = (np.floor(lo) != np.floor(hi)) & (hi < m - 1)                           # (the last cell is clamped)
        edge |= cell_line & (lo >= 0)
    ix = np.clip(np.floor(np.where(inside, fx.v, 0)), 0, nx - 2).astype(np.int64)
    iy = np.clip(np.floor(np.where(inside, fy.v, 0)), 0, ny - 2).astype(np.int64)
    hfl = np.asarray(hf, np.float32).reshape(-1).astype(np.float64)
    at = lambda i, j: TV(hfl[j * pitch + i])
    z00, z10, z01, z11 = at(ix, iy), at(ix + 1, iy), at(ix, iy + 1), at(ix + 1, iy + 1)
    tx, ty = fx - TV(ix.astype(np.float64)), fy - TV(iy.astype(np.float64))
    d1, d2 = z10 - z00, z11 - z01
    za, zb = fm(d1, tx, z00), fm(d2, tx, z01)
    dz = zb - za
    z = fm(dz, ty, za)
    gx = fm(d2 - d1, ty, d1) * inv
    gy = dz * inv
    ninv = tv_recip(tv_sqrt(fm(gx, gx, fm(gy, gy, TV(np.ones(shape))))))
    n = [-(gx * ninv), -(gy * ninv), ninv]
    out_z = const(cfg.hf_outside_z, shape)
    pick = lambda a, b: TV(np.where(inside, a.v, b.v), np.where(inside, a.e, b.e))
    return pick(z, out_z), [pick(a, b) for a, b in zip(n, up)], edge


def suspension_ref(cfg, st, hf=None):
    """fp64 restatement of wl_suspension_kernel on the state groups st [16, n, 4] with its rounding bound.  Returns a dict of
    TV pos, vel, comp [n, 4] and the mask `branch` of wheels left out of the fp64 check."""
    st = np.asarray(st, np.float32)
    n = st.shape[1]
    g = lambda grp, k: TV(st[grp, :, k].astype(np.float64)[:, None] * np.ones((1, 4)))
    p = [g(G_POS, k) for k in range(3)]
    w_, x_, y_, z_ = (g(G_QUAT, k) for k in range(4))
    v = [g(G_LINVEL, k) for k in range(3)]
    om = [g(G_ANGVEL, k) for k in range(3)]
    shape = (n, 4)
    R = rotmat(w_, x_, y_, z_)
    com = [const(cfg.com[k], shape) for k in range(3)]
    cw = rot(R, com)
    pc = [p[k] + cw[k] for k in range(3)]
    vb, wb = rotT(R, v), rotT(R, om)
    hx = np.array([cfg.hub_x_rear, cfg.hub_x_rear, cfg.hub_x_front, cfg.hub_x_front], np.float32).astype(np.float64)
    hy = float(np.float32(cfg.hub_y)) * np.array([1.0, -1.0, 1.0, -1.0])
    rho = [TV(np.broadcast_to(hx, shape)) - com[0], TV(np.broadcast_to(hy, shape)) - com[1], const(cfg.hub_z, shape) - com[2]]
    hub = rot(R, rho)
    hub = [hub[k] + pc[k] for k in range(3)]
    zt, nw, edge = _terrain(cfg, hf, hub[0], hub[1])
    r = const(cfg.wheel_radius, shape)
    comp = fm(-(hub[2] - zt), nw[2], r)
    nb = rotT(R, nw)
    rc = [fm(-r, nb[k], rho[k]) for k in range(3)]
    vc = cross(wb, rc)
    vc = [vc[k] + vb[k] for k in range(3)]
    tr = float(np.float32(cfg.susp_travel))
    pos = TV(np.clip(comp.v, -tr, tr), comp.e)
    sv = -dot3(nb, vc)
    touch = comp.v > 0
    vel = TV(np.where(touch, sv.v, 0.0), np.where(touch, sv.e, 0.0))
    branch = edge | (np.abs(comp.v) <= comp.e) | (np.abs(np.abs(comp.v) - tr) <= comp.e)
    return {"pos": pos, "vel": vel, "comp": comp, "branch": branch, "hub_z": hub[2], "n_z": nw[2]}


def check_fp64(got_pos, got_vel, ref, o64, what, min_kept=0.5):
    """|got - fp64| <= bound on every wheel off a branch edge; the fp64 oracle's outputs are rounded to fp32, so it is first
    checked against the restatement's value (within that rounding), and the comparison adds that rounding.  Returns the
    largest |err| / bound."""
    keep = ~ref["branch"]
    assert keep.mean() > min_kept, f"{what}: {int((~keep).sum())} of {keep.size} wheels on a branch edge"
    worst = 0.0
    for name, got, tv, o in (("pos", got_pos, ref["pos"], o64[0]), ("vel", got_vel, ref["vel"], o64[1])):
        o = np.asarray(o, np.float64)
        assert (np.abs(o - tv.v)[keep] <= U * np.abs(tv.v[keep]) + 1e-30).all(), f"{what}: {name}: fp64 oracle != restatement"
        bound = tv.e + U * np.abs(o)
        err = np.abs(np.asarray(got, np.float64) - o)
        ratio = np.where(keep, err / np.where(bound > 0, bound, 1.0), 0.0)
        i = np.unravel_index(np.argmax(ratio), ratio.shape)
        assert ratio[i] <= 1.0, f"{what}: {name} env {i[0]} wheel {i[1]}: |err| {err[i]:.3g} > bound {bound[i]:.3g}"
        assert (err[keep & (bound == 0)] == 0).all()
        worst = max(worst, float(ratio.max()))
    print(f"{what}: largest |err| / bound {worst:.3g} ({int(keep.sum())} of {keep.size} wheels, {int((~keep).sum())} on a branch edge)")
    return worst


# ---- specs, oracles and placed states ----------------------------------------------------------------------------------
def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def make_spec(task, n, seed=3, **kw):
    import wheeledlab_b200 as wl
    if task == "elevation":
        return wl.elevation_task(num_envs=n, seed=seed, **kw)
    if task == "visual":
        return wl.visual_task(num_envs=n, seed=seed, **kw)
    return wl.make_task(task, num_envs=n, seed=seed, **kw)


def oracles(spec):
    hf = spec.heightfield if int(spec.cfg.task) != 0 else None
    o32 = O.Oracle(spec.cfg, heightfield=hf, threads=8)
    o64 = O.Oracle(spec.cfg, heightfield=hf, kind="f64")
    o32.startup(); o32.reset(None, 0)
    return o32, o64


def both(o32, o64, st):
    o32.import_state(st); o64.import_state(st)
    return o32.suspension(), o64.suspension()


def quat_x(phi):
    return (math.cos(phi / 2), math.sin(phi / 2), 0.0, 0.0)


def quat_y(theta):
    return (math.cos(theta / 2), 0.0, math.sin(theta / 2), 0.0)


def place(st, k, p=None, q=None, v=None, w=None):
    if p is not None:
        st[G_POS, k, :3] = p
    if q is not None:
        st[G_QUAT, k] = q
    if v is not None:
        st[G_LINVEL, k, :3] = v
    if w is not None:
        st[G_ANGVEL, k, :3] = w


def hub_body(cfg):
    """Hub positions in the body (root) frame, [bl, br, fl, fr] x (x, y, z), fp64 of the fp32 constants."""
    f = lambda a: float(np.float32(a))
    return np.array([[f(cfg.hub_x_rear), f(cfg.hub_y), f(cfg.hub_z)], [f(cfg.hub_x_rear), -f(cfg.hub_y), f(cfg.hub_z)],
                     [f(cfg.hub_x_front), f(cfg.hub_y), f(cfg.hub_z)], [f(cfg.hub_x_front), -f(cfg.hub_y), f(cfg.hub_z)]])


def closed_form(cfg, st):
    """Flat ground: comp = r - hub_z(world), vel = -d(hub_z)/dt = -(v + w x R rho)_z while comp > 0, for states whose
    rotation is the exact rotation of the stored quaternion's angle.  Returns (pos, vel, slack): slack bounds what the
    stored quaternion's |q|^2 != 1 moves (rotmat(q) = |q|^2 R(q/|q|) + (1 - |q|^2) I)."""
    st = np.asarray(st, np.float64)
    q = st[G_QUAT]
    qn = q / np.linalg.norm(q, axis=1, keepdims=True)
    w, x, y, z = qn.T
    R = np.stack([1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y),
                  2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x),
                  2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)], axis=1).reshape(-1, 3, 3)
    hb = hub_body(cfg)
    com = np.array([float(np.float32(c)) for c in cfg.com])
    r, tr = float(np.float32(cfg.wheel_radius)), float(np.float32(cfg.susp_travel))
    hub_w = st[G_POS, :, None, :3] + np.einsum("nij,wj->nwi", R, hb)
    comp = r - hub_w[..., 2]
    arm = np.einsum("nij,wj->nwi", R, hb - com)                    # hub relative to the COM, world frame
    vz = st[G_LINVEL, :, None, 2] + np.cross(st[G_ANGVEL, :, None, :3], arm)[..., 2]
    delta = np.abs((q * q).sum(axis=1) - 1.0)[:, None]
    vmag = np.linalg.norm(st[G_LINVEL, :, :3], axis=1)[:, None] + np.linalg.norm(st[G_ANGVEL, :, :3], axis=1)[:, None] * (
        np.linalg.norm(hb - com, axis=1)[None, :] + r)
    slack_pos = 2 * delta * np.linalg.norm(hb, axis=1)[None, :]
    slack_vel = 8 * delta * vmag
    return np.clip(comp, -tr, tr), np.where(comp > 0, -vz, 0.0), comp, slack_pos, slack_vel


def closed_form_states(cfg, st, seed=0):
    """Placed flat-ground states for env k of st (at least 48 envs): level at a chosen compression (every 4th env lifted
    clear or pressed past +travel), rolled and pitched by +-1.5 and 12 deg, each with a prescribed v and w."""
    st = np.array(st, np.float32, copy=True)
    rng = np.random.default_rng(seed)
    r, hz = float(np.float32(cfg.wheel_radius)), float(np.float32(cfg.hub_z))
    comps = [0.004, 0.0005, -0.003, 0.015, 0.0099, -0.02, 0.001, 0.0]
    quats = [(1.0, 0.0, 0.0, 0.0)] + [f(math.radians(d)) for f in (quat_x, quat_y) for d in (1.5, -1.5, 12.0, -12.0)]
    for k in range(48):
        place(st, k, p=(0.1 * k, -0.2 * k, r - hz - comps[k % 8]), q=quats[(k // 8) % len(quats)] if k >= 8 else quats[0],
              v=tuple(rng.uniform(-2, 2, 3)), w=tuple(rng.uniform(-3, 3, 3)))
    return st


def check_closed_form(cfg, st, got, ref, what, tol64=False):
    """got = (pos, vel) of one build; within the restatement's bound (fp32) or the fp64 output rounding (fp64) plus the
    quaternion slack of the closed form."""
    pos_c, vel_c, comp_c, sp, sv = closed_form(cfg, st)
    for name, g, c, tv, slack in (("pos", got[0], pos_c, ref["pos"], sp), ("vel", got[1], vel_c, ref["vel"], sv)):
        bound = (U * np.abs(c) if tol64 else tv.e + U * np.abs(c)) + slack + 1e-15
        err = np.abs(np.asarray(g, np.float64) - c)
        if name == "vel":                                      # comp within its bound of 0: either side of the select
            err = np.where(np.abs(comp_c) <= ref["comp"].e, 0.0, err)
        assert (err <= bound).all(), f"{what}: {name} {g[err > bound][:4]} != closed form {c[err > bound][:4]}"
    return comp_c


# ---- 1. closed-form placed states ----------------------------------------------------------------------------------------
@pytest.fixture(scope="module", params=["drift", "f1tenth_drift"])
def flat(request):
    spec = make_spec(request.param, 64)
    o32, o64 = oracles(spec)
    return spec, o32, o64


def _run_placed(spec, o32, o64, st, what):
    (p32, v32), (p64, v64) = both(o32, o64, st)
    ref = suspension_ref(spec.cfg, st)
    check_closed_form(spec.cfg, st, (p32, v32), ref, f"{what} fp32")
    check_closed_form(spec.cfg, st, (p64, v64), ref, f"{what} fp64", tol64=True)
    return p32, v32, p64, v64


def test_level_chassis_gives_the_chosen_compression_on_every_wheel(flat):
    spec, o32, o64 = flat
    c = spec.cfg
    st = o32.export_state()
    r, hz = float(np.float32(c.wheel_radius)), float(np.float32(c.hub_z))
    tr = float(np.float32(c.susp_travel))
    comps = [0.004, 0.0005, -0.003, 0.0099, 0.015, -0.02, 0.0, 0.001] * 2
    for k, cm in enumerate(comps):
        place(st, k, p=(0.3 * k, -0.1 * k, r - hz - cm), q=(1.0, 0.0, 0.0, 0.0), v=(0.0, 0.0, 0.0), w=(0.0, 0.0, 0.0))
    p32, v32, p64, v64 = (x[:16] for x in _run_placed(spec, o32, o64, st, "level"))
    want = np.clip(np.array(comps), -tr, tr)[:, None] * np.ones((1, 4))
    assert np.allclose(p64, want, rtol=0, atol=2e-8)                          # the chosen compression, every wheel
    assert (p32[5] == np.float32(-c.susp_travel)).all() and (v32[5] == 0).all()  # lifted clear: -travel, exactly 0
    assert (p32[4] == np.float32(c.susp_travel)).all()                         # beyond +travel: +travel
    assert (v32 == 0).all() and (v64 == 0).all()                               # at rest


@pytest.mark.parametrize("axis", ["roll", "pitch"])
@pytest.mark.parametrize("deg", [1.5, -1.2, 20.0])
def test_rolled_or_pitched_chassis_splits_left_right_or_front_rear(flat, axis, deg):
    """R_x(a) raises the left (+hub_y) hubs by 2 hub_y sin a against the right; R_y(a) lowers the front hubs by
    (hub_x_front - hub_x_rear) sin a against the rear.  At 20 deg one side hangs clear (-travel) and the other is pressed
    past +travel."""
    spec, o32, o64 = flat
    c = spec.cfg
    st = o32.export_state()
    a = math.radians(deg)
    q = quat_x(a) if axis == "roll" else quat_y(a)
    hb = hub_body(c)
    r, tr = float(np.float32(c.wheel_radius)), float(np.float32(c.susp_travel))
    zc = hb[0, 2] * math.cos(a) - (float(np.mean(hb[:, 0])) * math.sin(a) if axis == "pitch" else 0.0)   # mean hub height
    for k in range(16):
        place(st, k, p=(0.1 * k, 0.05 * k, r - zc - 0.001 - 0.0001 * k), q=q, v=(0.0, 0.0, 0.0), w=(0.0, 0.0, 0.0))
    p32, v32, p64, v64 = (x[:16] for x in _run_placed(spec, o32, o64, st, f"{axis} {deg}"))
    if axis == "roll":
        low, high, d_want = [1, 3], [0, 2], 2 * hb[0, 1] * math.sin(a)          # right minus left compression
    else:
        low, high, d_want = [2, 3], [0, 1], (hb[2, 0] - hb[0, 0]) * math.sin(a)  # front minus rear compression
    for pos in (p32.astype(np.float64), p64.astype(np.float64)):
        if abs(deg) < 10:
            assert (np.abs(pos) < tr).all()
            assert np.allclose(pos[:, low] - pos[:, high], d_want, rtol=0, atol=1e-6)
        else:
            assert (pos[:, high] == np.float32(-tr)).all() and (pos[:, low] == np.float32(tr)).all()
    assert (v32 == 0).all() and (v64 == 0).all()


def test_prescribed_velocity_gives_the_compression_rate_of_each_wheel(flat):
    """vel = -(v + w x R rho)_z on every touching wheel; the wheels a roll lifts clear report exactly 0."""
    spec, o32, o64 = flat
    c = spec.cfg
    st = o32.export_state()
    r, hz = float(np.float32(c.wheel_radius)), float(np.float32(c.hub_z))
    rng = np.random.default_rng(1)
    for k in range(16):
        q = (1.0, 0.0, 0.0, 0.0) if k < 8 else quat_x(math.radians(12.0 if k % 2 else -12.0))
        place(st, k, p=(0.0, 0.0, r - hz - 0.003), q=q, v=tuple(rng.uniform(-2, 2, 3)), w=tuple(rng.uniform(-3, 3, 3)))
    place(st, 0, v=(0.0, 0.0, -0.5), w=(0.0, 0.0, 0.0))                          # sinking at 0.5 m/s: +0.5 on every wheel
    place(st, 1, v=(0.0, 0.0, 0.0), w=(1.0, 0.0, 0.0))                           # rolling right side down: vel = -w_x rho_y
    place(st, 2, v=(0.0, 0.0, 0.0), w=(0.0, 1.0, 0.0))                           # pitching nose down: vel = +w_y rho_x
    p32, v32, p64, v64 = (x[:16] for x in _run_placed(spec, o32, o64, st, "velocity"))
    hb, com = hub_body(c), np.array([float(np.float32(x)) for x in c.com])
    rho = hb - com
    assert np.allclose(v64[0], 0.5, rtol=0, atol=1e-7)
    assert np.allclose(v64[1], -rho[:, 1], rtol=0, atol=1e-7) and v64[1, 1] > 0 > v64[1, 0]
    assert np.allclose(v64[2], rho[:, 0], rtol=0, atol=1e-7) and v64[2, 2] > 0 > v64[2, 0]
    lifted = p32[8:] == np.float32(-c.susp_travel)
    assert lifted.any() and (v32[8:][lifted] == 0).all() and (v64[8:][p64[8:] <= 0] == 0).all()


def test_mixed_closed_form_states(flat):
    """The placed states the GPU test loads into the kernel, checked here on both oracle builds."""
    spec, o32, o64 = flat
    st = closed_form_states(spec.cfg, o32.export_state())
    p32, v32, p64, v64 = _run_placed(spec, o32, o64, st, "mixed")
    tr = np.float32(spec.cfg.susp_travel)
    assert (p32 == -tr).any() and (p32 == tr).any() and ((np.abs(p32) < tr) & (v32 != 0)).any()


def test_wheel_order_is_bl_br_fl_fr():
    """One wheel pressed 6 mm deeper than the others by a pure pitch + roll that lowers exactly that corner."""
    spec = make_spec("drift", 4)
    o32, o64 = oracles(spec)
    st = o32.export_state()
    c = spec.cfg
    r, hz = float(np.float32(c.wheel_radius)), float(np.float32(c.hub_z))
    for k, (sx, sy) in enumerate([(-1, 1), (-1, -1), (1, 1), (1, -1)]):           # bl, br, fl, fr: the corner to lower
        q = np.array(quat_y(math.radians(2.0) * sx)) + 0.0
        qr = np.array(quat_x(math.radians(-2.0) * sy))
        w1, x1, y1, z1 = qr
        w2, x2, y2, z2 = q
        qq = (w1 * w2 - x1 * x2 - y1 * y2 - z1 * z2, w1 * x2 + x1 * w2 + y1 * z2 - z1 * y2,
              w1 * y2 - x1 * z2 + y1 * w2 + z1 * x2, w1 * z2 + x1 * y2 - y1 * x2 + z1 * w2)
        place(st, k, p=(0.0, 0.0, r - hz - 0.002), q=qq, v=(0.0,) * 3, w=(0.0,) * 3)
    (p32, _), (p64, _) = both(o32, o64, st)
    assert (np.argmax(p32, axis=1) == np.arange(4)).all() and (np.argmax(p64, axis=1) == np.arange(4)).all()


# ---- 2. fp32 oracle against fp64 oracle on rollout states ------------------------------------------------------------------
def rollout_state(spec, o32, t0, steps):
    """The fp32 oracle's state after steps t0 .. t0 + steps - 1 with synth_actions.  Before the first, every third env is put
    3 steps before its time-out, so auto-resets are among the states."""
    if t0 == 0:
        st = o32.export_state()
        ep = st[G_POS, :, 3].view(np.int32).copy()
        ep[::3] = int(spec.cfg.max_episode_length) - 3
        st[G_POS, :, 3] = ep.view(np.float32)
        o32.import_state(st)
    for t in range(t0, t0 + steps):
        o32.step(o32.synth_actions(t, dist=t % 2), t)
    return o32.export_state()


@pytest.mark.parametrize("task", TASKS)
def test_fp32_oracle_is_within_the_bound_of_fp64_on_rollouts(task):
    spec = make_spec(task, 96)
    o32, o64 = oracles(spec)
    hf = spec.heightfield if task == "elevation" else None
    for t0, steps in ((0, 0), (0, 5), (5, 7)):
        st = rollout_state(spec, o32, t0, steps)
        (p32, v32), (p64, v64) = both(o32, o64, st)
        ref = suspension_ref(spec.cfg, st, hf)
        assert check_fp64(p32, v32, ref, (p64, v64), f"{task} after {t0 + steps} steps") <= 1.0
        assert (np.abs(p32) <= np.float32(spec.cfg.susp_travel)).all()
        assert (v32[ref["comp"].v < -ref["comp"].e] == 0).all()
        # a zero vel keeps the sign of the negated dot product (-0 for a resting wheel on a flat cell), as the kernel's does
        zero = (v32 == 0) & (ref["vel"].v == 0)
        assert (np.signbit(v32[zero]) == np.signbit(ref["vel"].v[zero])).all() and (_bits(v32) == _bits(v64))[zero].all()


def test_restatement_bound_is_not_vacuous():
    """The bound sits within 2^10 of the error it bounds on the Elevation rollout: a bound that large would pass a kernel
    that is wrong by far more than its rounding."""
    spec = make_spec("elevation", 96)
    o32, o64 = oracles(spec)
    st = rollout_state(spec, o32, 0, 7)
    (p32, v32), (p64, v64) = both(o32, o64, st)
    ref = suspension_ref(spec.cfg, st, spec.heightfield)
    keep = ~ref["branch"] & (ref["comp"].v > 0)
    rel = ref["vel"].e[keep] / np.maximum(np.abs(ref["vel"].v[keep]), 1e-3)
    assert np.median(rel) < 2 ** 10 * U
    assert check_fp64(p32, v32, ref, (p64, v64), "elevation bound") > 0.0
