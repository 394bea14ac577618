"""The Visual task's camera term (wl_camera_kernel) at every camera geometry wl_create accepts, not only the task's own
80 x 60 frame (80 x 40 kept pixels).  wl_create takes a width W that is a multiple of 4 from 4 to 128, 3 to 64 kept rows
(vis_cam_h - vis_cam_row0) and at most WL_CAM_MAX_PIXELS = 4096 pixels; compat lowers any TiledCameraCfg width / height into
those fields.  The kernel's indexing depends on the geometry: W4 = W / 4 column groups, RG = 128 / W4 row groups (threads
at or above RG * W4 idle), the reflected border columns and rows, the mask Jp (row stride W + 8) and the horizontal pass
Hp (rows + 4 padded rows) in fixed shared arrays, the column / row tables, the proprioceptive float4 at offset W * rows of
an 8 + W * rows row, and the white fraction n_white / npix that feeds the contrast op.  GEOMETRIES says which edge each case
reaches.

GPU, every geometry:
- In raw and aug mode at N = 1, 33 and 1000, with a third of the envs 3 steps before their time-out: wl_observe before
  the first step, 8 steps alternating wl_step (quad and thread-per-env) with the staged step, wl_camera with drawn and
  with explicit parameters -- the camera floats and the proprioceptive floats of every row bit for bit against the CPU
  oracle; reward, done masks, episode log, final state and reward weights as test_elev_visual_coverage_gpu checks them.
  wl_camera must leave the 8 proprioceptive floats of a row alone.
- The rendered white mask against a plain fp64 ray / plane / mesh-cell restatement at placed poses; a pixel may differ only
  where fp32 cannot decide it (_render64 states the bound), and every other mismatch is named.
- The aug-mode output against an fp64 restatement of torchvision's ColorJitter / GaussianBlur / Grayscale / Normalize on
  the kernel's own mask, within 2e-6.
- wl_rollout still refuses a camera handle.

The edges of what is accepted: wl_create refuses the geometries just outside (and compat's env construction with it); the
device policy drives the widest row it takes (8 + 120 x 34 = 4088 floats) against the oracle, and wl_policy_act,
wl_actor_mean and wl_ppo_update_wide refuse rows of 4100 and 4104 floats without writing anything.

The CPU tests pin the oracle itself away from 80 x 40 (its render and post-processing against the same fp64 restatements
at every geometry), pin the fp64 post-processing to the torchvision golden vectors, check that compat lowers a camera to the
same wl_config as the helper here, and check wl_create's geometry verdicts without a device.

The file takes about 31 s on one H100 80GB HBM3 (power limit 400 W), most of it in the CPU oracle."""
import ctypes as C
import math
import sys
from pathlib import Path

import numpy as np
import pytest

import oracle_lib as O
import test_elev_visual_coverage_gpu as ev

torch = pytest.importorskip("torch")

ROOT = Path(__file__).resolve().parent.parent
DEV = "cuda:0"
FOCAL, H_AP, V_AP = 1.9299999475479126, 3.8959999084472656, 2.453000068664551   # TiledCameraCfg.spawn of the Visual task
U = 2.0 ** -24                                              # fp32 unit roundoff
SENTINEL = np.uint32(0x7FC0DEAD)                            # a NaN payload no kernel writes

# name: (W, H, row0) -- row0 None is H // 3, as compat sets it.  W4 = W / 4, RG = 128 // W4 (row groups), idle threads
# 128 - RG * W4.  Jp holds rows * (W + 8) bytes of 4096 + 8 * 64 = 4608; Hp holds (rows + 4) * W floats of 4096 + 4 * 128.
GEOMETRIES = {
    "4x3": (4, 4, None),             # W4 1, RG 128: one column group; the smallest reflect (columns 1, 2 / rows 1, 2 of 3)
    "4x64": (4, 96, None),           # W4 1, RG 128: the most kept rows; yo_s full; reflected border written by 64 threads
    "12x5": (12, 7, None),           # W4 3, RG 42: W4 does not divide 128, 2 idle threads
    "44x63": (44, 94, None),         # W4 11, RG 11: 7 idle threads
    "84x48": (84, 72, None),         # W4 21, RG 6: 2 idle threads; wider than the task's 80
    "128x3": (128, 4, None),         # W4 32, RG 4: the widest; fewer rows than row groups (one group renders nothing)
    "64x64": (64, 96, None),         # Jp at the end of its shared array (64 x 72 = 4608 bytes); 4096 pixels
    "128x32": (128, 48, None),       # Hp at the end of its shared array (36 x 128 = 4608 floats); 4096 pixels; obs row 4104
    "120x34": (120, 51, None),       # 4080 pixels: obs row 4088, the widest the device policy takes
    "124x33": (124, 49, None),       # W4 31, RG 4, 4 idle threads; 4092 pixels: obs row 4100
    "8x3_row0_0": (8, 3, 0),         # the whole frame kept (row0 = 0): a row0 the H // 3 rule cannot give
    "80x40": (80, 60, None),         # the task's own camera (W4 20, RG 6, 8 idle threads): the control
}
# explicit ColorJitter / blur parameters (brightness, contrast, saturation, hue, sigma, op order): sigma at both ends of the
# task's (0.1, 5.0) and five op orders
AUGS = np.array([
    [0.4, 0.85, 1.5, 0.1, 0.1, 0, 1, 2, 3],
    [1.6, 1.2, 0.3, -0.2, 5.0, 3, 1, 0, 2],
    [0.9, 0.8, 1.0, 0.0, 1.3, 2, 3, 1, 0],
    [1.3, 1.1, 0.6, 0.4, 5.0, 1, 0, 3, 2],
    [0.7, 0.9, 1.8, 0.3, 0.1, 1, 2, 0, 3],
], np.float32)


def _geometry(name):
    W, H, r0 = GEOMETRIES[name]
    return W, H, H // 3 if r0 is None else r0


def _map(seed):
    """A 500 x 500 traversability map of independent random cells: neighbouring cells differ half the time, so a pixel
    rendered from the wrong column, row or ray shows."""
    return np.random.default_rng(seed).random((500, 500)) < 0.5


def cam_spec(W, H, row0=None, n=1, camera="aug", seed=7, traversability=None, **kw):
    """visual_task with a W x H camera keeping rows row0.. (default H // 3), set the way compat lowers a TiledCameraCfg."""
    import wheeledlab_b200 as wl
    spec = wl.visual_task(num_envs=n, seed=seed, camera=camera, traversability=traversability, **kw)
    c = spec.cfg
    c.vis_cam_w, c.vis_cam_h = W, H
    c.vis_cam_row0 = H // 3 if row0 is None else row0
    c.vis_cam_fx, c.vis_cam_fy = FOCAL * W / H_AP, FOCAL * H / V_AP
    c.vis_cam_cx, c.vis_cam_cy = W / 2.0, H / 2.0
    spec.obs_dim = 8 + W * (H - c.vis_cam_row0)
    return spec


def _spec(name, n, camera="aug", seed=7, **kw):
    W, H, r0 = _geometry(name)
    return cam_spec(W, H, r0, n=n, camera=camera, seed=seed, **kw)


def _npix(spec):
    c = spec.cfg
    return int(c.vis_cam_w) * (int(c.vis_cam_h) - int(c.vis_cam_row0))


def _sentinel(n, d):
    return torch.from_numpy(np.full((n, d), SENTINEL, np.uint32).view(np.float32)).to(DEV)


def _check_camera_call(spec, got, ref, what):
    """wl_camera into a sentinel-filled buffer: the camera floats equal the oracle's, the proprioceptive ones untouched."""
    k = _npix(spec)
    got = got.cpu().numpy()
    bad = np.flatnonzero((ev._bits(got[:, :k]) != ev._bits(ref[:, :k])).any(axis=1))
    assert bad.size == 0, f"{what}: camera differs at envs {bad[:8]} (max |diff| {np.nanmax(np.abs(got[:, :k] - ref[:, :k])):.3g})"
    assert (ev._bits(got[:, k:]) == SENTINEL).all(), f"{what}: wl_camera wrote into the proprioceptive floats"


# ---- placed poses and the fp64 restatements ---------------------------------------------------------------------------
def _poses():
    """(x, y, z, yaw, pitch, roll): level, pitched down and up, rolled, raised, and at the map's edge looking out."""
    rng = np.random.default_rng(3)
    out = [(1.0, -2.0, 0.0, 0.3, 0.0, 0.0), (-30.3, 40.7, 0.01, -2.0, 0.05, 0.0), (60.2, -81.9, 0.0, 1.1, -0.04, 0.0),
           (121.0, 3.0, 0.0, 0.0, 0.0, 0.0), (-10.0, 123.5, 0.5, 1.5707963, 0.2, 0.0), (20.5, 20.5, 2.0, 0.7, 0.6, 0.0),
           (-70.0, -70.0, 0.0, -0.9, 0.0, 0.25), (5.25, -5.25, 0.3, 2.9, 0.35, -0.15)]
    for _ in range(8):
        out.append((rng.uniform(-110, 110), rng.uniform(-110, 110), rng.choice([0.0, 0.1, 1.0]), rng.uniform(-math.pi, math.pi),
                    rng.uniform(-0.3, 0.5), rng.uniform(-0.2, 0.2)))
    return out


POSES = _poses()


def _qmul(a, b):
    w1, x1, y1, z1 = a
    w2, x2, y2, z2 = b
    return (w1 * w2 - x1 * x2 - y1 * y2 - z1 * z2, w1 * x2 + x1 * w2 + y1 * z2 - z1 * y2,
            w1 * y2 - x1 * z2 + y1 * w2 + z1 * x2, w1 * z2 + x1 * y2 - y1 * x2 + z1 * w2)


def _posed(state):
    """The state with env i's root at POSES[i]: q = q_z(yaw) q_y(pitch) q_x(roll), (w, x, y, z)."""
    st = state.copy()
    for i, (x, y, z, yaw, pitch, roll) in enumerate(POSES):
        q = _qmul(_qmul((math.cos(yaw / 2), 0.0, 0.0, math.sin(yaw / 2)), (math.cos(pitch / 2), 0.0, math.sin(pitch / 2), 0.0)),
                  (math.cos(roll / 2), math.sin(roll / 2), 0.0, 0.0))
        st[0, i, :3] = (x, y, z)
        st[1, i] = q
    return st


def _render64(c, state, trav):
    """fp64 pinhole camera: the ray through each kept pixel centre, d = R (1, -xo, -yo) (x forward, y left, z up), from
    pc = p + R cam_pos to the plane z = 0, then the mesh cell floor((h - x0) / dx) of the map; black outside the mesh, for
    rays that do not descend and beyond the 100 m clip.  Returns (white, doubt) [n, rows, W]: doubt marks the pixels whose
    colour fp32 cannot decide.

    The bound: in fp32 each component of d carries at most ~12 u s of error (u = 2^-24, s = 1 + |xo| + |yo|): the rotation
    matrix from the fp32 quaternion (<= 9 u per entry, three roundings), the two fmas of d and the division of xo, yo.  We
    take e_d = 16 u s, and for the camera centre pc = p + R cam the same 16 u per unit of |p_j| + |cam|_1 (e_z for z).  The
    depth tt = pc_z / -d_z then errs by e_t = tt (e_d / |d_z| + 4 u) + e_z / |d_z|, the hit point h = pc + tt d by
    e_h = |d_xy| e_t + tt e_d + e_xy + 4 u |h|, its cell coordinate by e_h + 4 u |h - x0| more (the fp32 inverse cell size,
    the difference and the product).  A pixel is in doubt if, with a factor 4 on each bound: its hit point lies within e_h
    (plus the cell term) of a cell edge, its depth within e_t of the 100 m clip, or |d_z| < e_d (the ray is that close to
    horizontal).  Everything else fp32 must get right."""
    W, H, r0 = int(c.vis_cam_w), int(c.vis_cam_h), int(c.vis_cam_row0)
    u, v = np.meshgrid(np.arange(W, dtype=np.float64), np.arange(r0, H, dtype=np.float64))
    xo = (u + 0.5 - c.vis_cam_cx) / c.vis_cam_fx
    yo = (v + 0.5 - c.vis_cam_cy) / c.vis_cam_fy
    cam = np.array(list(c.vis_cam_pos), np.float64)
    x0, y0, dx, dy = (float(getattr(c, k)) for k in ("vis_mesh_x0", "vis_mesh_y0", "vis_mesh_dx", "vis_mesh_dy"))
    ncol, nrow = int(c.vis_cols), int(c.vis_rows)
    e_d = 16 * U * (1 + np.abs(xo) + np.abs(yo))
    K = 4.0
    whites, doubts = [], []
    for i in range(int(c.num_envs)):
        p = state[0, i, :3].astype(np.float64)
        w, x, y, z = state[1, i].astype(np.float64)
        R = np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                      [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                      [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])
        pc = p + R @ cam
        d = R[:, 0] - xo[..., None] * R[:, 1] - yo[..., None] * R[:, 2]
        dz = d[..., 2]
        with np.errstate(divide="ignore", invalid="ignore"):
            tt = pc[2] / -dz
            hx, hy = pc[0] + tt * d[..., 0], pc[1] + tt * d[..., 1]
            qx, qy = (hx - x0) / dx, (hy - y0) / dy
            fx, fy = np.floor(qx), np.floor(qy)
            hit = (dz < 0) & (pc[2] > 0) & (tt <= 100.0)
            inside = hit & (fx >= 0) & (fy >= 0) & (fx < ncol - 1) & (fy < nrow - 1)
            white = np.zeros(dz.shape, bool)
            white[inside] = trav[fy[inside].astype(np.int64), fx[inside].astype(np.int64)]
            adz = np.abs(dz)
            e_z, e_xy = 16 * U * (abs(p[2]) + np.abs(cam).sum()), 16 * U * (np.abs(p[:2]).max() + np.abs(cam).sum())
            e_t = tt * (e_d / adz + 4 * U) + e_z / adz
            e_h = np.maximum(np.abs(d[..., 0]), np.abs(d[..., 1])) * e_t + tt * e_d + e_xy + 4 * U * np.maximum(np.abs(hx), np.abs(hy))
            edge = np.minimum(np.abs(qx - np.round(qx)) * dx, np.abs(qy - np.round(qy)) * dy)
            near_edge = (dz < 0) & (tt <= 100.0 + K * e_t) & (edge < K * (e_h + 4 * U * np.maximum(np.abs(hx - x0), np.abs(hy - y0))))
            doubt = near_edge | ((dz < 0) & (np.abs(tt - 100.0) < K * e_t)) | (adz < K * e_d)
        whites.append(white)
        doubts.append(doubt)
    return np.stack(whites), np.stack(doubts)


def _check_render(c, state, trav, got, what):
    """got [n, rows, W] bool against _render64: every mismatch outside the doubt set is named."""
    exp, doubt = _render64(c, state, trav)
    bad = np.argwhere((got != exp) & ~doubt)
    msg = "; ".join(f"env {i} row {r} col {k}: got {int(got[i, r, k])}" for i, r, k in bad[:12])
    assert bad.shape[0] == 0, f"{what}: {bad.shape[0]} pixels differ from the fp64 render where fp32 decides them: {msg}"
    assert doubt.mean() < 0.05, f"{what}: {doubt.mean():.1%} of the pixels are in doubt: the bound decides too little"
    assert 0.05 < exp.mean() < 0.95, f"{what}: the placed poses see a blank frame (white fraction {exp.mean():.3f})"
    return int(((got != exp) & doubt).sum())


GRAY = 0.2989 + 0.587 + 0.114                              # torchvision rgb_to_grayscale of a grey pixel v is GRAY * v


def _post64(W, rows, white, aug):
    """camera_data_rgb_flattened[_aug] in fp64 on masks [n, rows * W] (aug None: raw).  The two-colour frame stays two-valued
    under ColorJitter, applied in the given op order to the class values (v0, v1) = (0, 1): brightness scales and clamps;
    contrast blends toward the frame's mean grey, p GRAY v1 + (1 - p) GRAY v0 with p the white fraction, and clamps;
    saturation blends toward the pixel's own grey GRAY v (torchvision's weights sum to 0.9999, so this moves a grey by
    (1 - s) 1e-4 v) and clamps; hue leaves a grey pixel unchanged.  Then torchvision's 5-tap Gaussian kernel
    exp(-x^2 / 2 sigma^2), x = -2..2, normalised, applied along rows and columns with reflect padding (numpy's "reflect",
    which does not repeat the edge pixel), Grayscale and (x - 0.5) / 0.5."""
    m = np.asarray(white, bool).reshape(-1, rows, W)
    if aug is None:
        return ((m * GRAY - 0.5) / 0.5).reshape(m.shape[0], -1)
    b, ct, sa, _, sigma = (float(x) for x in aug[:5])
    x = np.arange(-2, 3, dtype=np.float64)
    k = np.exp(-0.5 * (x / sigma) ** 2)
    k /= k.sum()
    out = []
    for f in m:
        p, v0, v1 = f.mean(), 0.0, 1.0
        for op in np.asarray(aug[5:9]).astype(int):
            if op == 0:
                v0, v1 = np.clip(b * v0, 0, 1), np.clip(b * v1, 0, 1)
            elif op == 1:
                mean = p * GRAY * v1 + (1 - p) * GRAY * v0
                v0, v1 = np.clip(ct * v0 + (1 - ct) * mean, 0, 1), np.clip(ct * v1 + (1 - ct) * mean, 0, 1)
            elif op == 2:
                v0, v1 = np.clip(sa * v0 + (1 - sa) * GRAY * v0, 0, 1), np.clip(sa * v1 + (1 - sa) * GRAY * v1, 0, 1)
        img = np.pad(np.where(f, v1, v0), 2, mode="reflect")
        hz = sum(k[j] * img[:, j:j + W] for j in range(5))
        bl = sum(k[j] * hz[j:j + rows, :] for j in range(5))
        out.append(((GRAY * bl - 0.5) / 0.5).reshape(-1))
    return np.stack(out)


def _masks(W, rows, seed):
    """Masks of one geometry: all black, all white, a lower band, random pixels, random blocks, stripes."""
    rng = np.random.default_rng(seed)
    m = np.zeros((6, rows, W), bool)
    m[1] = True
    m[2, rows // 2:] = True
    m[3] = rng.random((rows, W)) < 0.4
    for _ in range(4):
        r, k = rng.integers(0, rows), rng.integers(0, W)
        m[4, r:r + rng.integers(1, 9), k:k + rng.integers(1, 17)] = True
    m[5, :, ::3] = True
    return m.reshape(6, -1).astype(np.uint8)


# ---- 1. the kernel against the oracle, bit for bit ---------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 33, 1000])
@pytest.mark.parametrize("mode", ["raw", "aug"])
@pytest.mark.parametrize("geom", list(GEOMETRIES))
def test_camera_geometry_matches_oracle(geom, mode, n):
    ev._need_gpu()
    spec = _spec(geom, n, mode, seed=7, traversability=_map(7))
    sim, orc = ev._pair(spec)
    D, what0 = spec.obs_dim, f"{geom} {mode} n={n}"
    assert sim.obs_dim == orc.obs_dim == D
    ev._near_timeout(sim, orc)
    ev._check_obs(spec, sim.observe(0, 2).cpu().numpy(), orc.observe(0, 2), f"{what0}: observe before the first step")
    white = [orc.camera_render(i) for i in range(n)]
    n_done = 0
    for t in range(8):
        what = f"{what0} step {t}"
        act = sim.synth_actions(t)
        log = torch.empty(16, device=DEV)
        if t % 2:
            rew, bits = sim.step_stage_a(act, t)
            obs, term, trunc = sim.step_stage_b(bits, t, log=log)
            out = (obs, rew, term, trunc)
        else:
            sim.set_kernel_variant(4 if t % 4 == 0 else 1)    # the quad kernel, then thread-per-env
            out = sim.step(act, t, log=log)
        sim.flush_log()
        n_done += ev._check_step(spec, out, orc.step(act.cpu().numpy(), t), what)
        ev._check_log(spec, log, orc.log(), what)
        white += [orc.camera_render(i) for i in range(n)]
    _check_camera_call(spec, sim.camera(8, _sentinel(n, D)), orc.camera(8), f"{what0}: wl_camera, drawn parameters")
    for k, aug in enumerate(AUGS):
        got = sim.camera(9, _sentinel(n, D), torch.from_numpy(aug).to(DEV))
        _check_camera_call(spec, got, orc.camera(9, aug), f"{what0}: wl_camera, explicit parameters {k}")
    ev._check_end(sim, orc, what0)
    assert n_done > 0, f"{what0}: no env reset in the run"
    frac = float(np.mean(white))
    assert 0.0 < frac < 1.0, f"{what0}: blank frames (white fraction {frac})"


# ---- 2. the kernel against plain fp64 restatements ---------------------------------------------------------------------
def _posed_sims(geom, modes, seed=5):
    """One sim per camera mode, every env at its placed pose (the same state in each)."""
    import wheeledlab_b200 as wl
    trav = _map(seed)
    sims = []
    for mode in modes:
        sim = wl.WheeledSim(_spec(geom, len(POSES), mode, seed=seed, traversability=trav), DEV); sim.startup(); sim.reset(None, 0)
        sims.append(sim)
    st = _posed(sims[0].groups.cpu().numpy())
    for sim in sims:
        sim.groups.copy_(torch.from_numpy(st))
    return sims, st, trav


def _gpu_mask(sim):
    """The white mask off the raw-mode camera: every pixel must be exactly one of the two grey values."""
    spec = sim.spec
    k = _npix(spec)
    cam = sim.camera(0, torch.zeros((sim.num_envs, spec.obs_dim), device=DEV)).cpu().numpy()[:, :k]
    g0, g1 = O.camera_post(spec.cfg, np.array([[0] * k, [1] * k], np.uint8), None)[:, 0]
    bits = ev._bits(cam)
    assert ((bits == ev._bits(g0)) | (bits == ev._bits(g1))).all(), "a raw-mode pixel is neither grey value"
    return bits == ev._bits(g1)


@pytest.mark.gpu
@pytest.mark.parametrize("geom", list(GEOMETRIES))
def test_camera_render_matches_fp64(geom):
    ev._need_gpu()
    (sim,), st, trav = _posed_sims(geom, ["raw"])
    W, H, r0 = _geometry(geom)
    _check_render(sim.cfg, st, trav, _gpu_mask(sim).reshape(-1, H - r0, W), f"{geom}, GPU")


@pytest.mark.gpu
@pytest.mark.parametrize("geom", list(GEOMETRIES))
def test_camera_post_processing_matches_fp64(geom):
    """The aug-mode output for explicit parameters against _post64 on the raw-mode mask of the same state, within 2e-6 (the
    oracle's own tolerance against torchvision, test_golden_cpu)."""
    ev._need_gpu()
    (raw, aug), _, _ = _posed_sims(geom, ["raw", "aug"])
    W, H, r0 = _geometry(geom)
    k = W * (H - r0)
    mask = _gpu_mask(raw)
    assert 0 < mask.mean() < 1
    out = raw.camera(0, torch.zeros((raw.num_envs, k + 8), device=DEV)).cpu().numpy()[:, :k]
    assert np.abs(out - _post64(W, H - r0, mask, None)).max() <= 1e-6
    for j, a in enumerate(AUGS):
        out = aug.camera(0, torch.zeros((aug.num_envs, k + 8), device=DEV), torch.from_numpy(a).to(DEV)).cpu().numpy()[:, :k]
        err = np.abs(out - _post64(W, H - r0, mask, a)).max()
        assert err <= 2e-6, f"{geom} parameters {j}: max |kernel - fp64| = {err:.3g}"


# ---- 3. the edges of what is accepted ----------------------------------------------------------------------------------
# (W, H, row0 or None, fx or None): just outside what wl_create takes
REFUSED = {
    "W0": (0, 60, None, None), "W2": (2, 60, None, None), "W6": (6, 60, None, None), "W132": (132, 45, None, None),
    "rows2": (80, 3, None, None), "rows65": (4, 97, None, None),
    "128x33": (128, 49, None, None), "100x41": (100, 61, None, None),     # 4224 and 4100 pixels
    "row0_neg": (80, 38, -2, None), "fx0": (80, 60, None, 0.0), "fx_neg": (80, 60, None, -57.0),
}


def _create_verdict(spec):
    """wl_create's message on spec without a device: the cfg also has dr_num_buckets = 0, which wl_create refuses after the
    camera checks and before it touches a device, so "dr_num_buckets" means the camera was accepted.  No handle may be left."""
    import wheeledlab_b200 as wl
    spec.cfg.dr_num_buckets = 0
    nbytes = int(wl.lib.wl_state_bytes(int(spec.cfg.num_envs)))
    state = np.zeros(nbytes + 256, np.uint8)
    aux = np.zeros(spec.heightfield.size + 16, np.uint8)
    h = C.c_void_p()
    rc = wl.lib.wl_create(C.byref(spec.cfg), C.c_void_p((state.ctypes.data + 255) & ~255), nbytes,
                          C.c_void_p((aux.ctypes.data + 15) & ~15), C.byref(h))
    assert rc != 0 and not h.value
    return wl.lib.wl_last_error().decode()


def test_wl_create_takes_every_geometry_and_refuses_the_ones_outside():
    small = np.ones((8, 8), bool)
    for name in GEOMETRIES:
        for mode in ("raw", "aug"):
            msg = _create_verdict(_spec(name, 4, mode, traversability=small))
            assert "dr_num_buckets" in msg, (name, mode, msg)
    for name, (W, H, r0, fx) in REFUSED.items():
        for mode in ("raw", "aug"):
            spec = cam_spec(W, H, r0, n=4, camera=mode, traversability=small)
            if fx is not None:
                spec.cfg.vis_cam_fx = fx
            assert "bad camera geometry" in _create_verdict(spec), (name, mode)


@pytest.mark.gpu
def test_env_construction_refuses_lowered_geometries_outside_the_limits(ref_registry):
    """compat lowers any TiledCameraCfg; building the env from one outside the limits fails with wl_create's message.  Every
    REFUSED case but the negative row0, which compat cannot produce (it keeps rows H // 3..); fx <= 0 is a focal length
    <= 0."""
    ev._need_gpu()
    import wheeledlab_b200 as wl
    from wheeledlab_b200.compat import env_from_reference_cfg
    for name, (W, H, r0, fx) in REFUSED.items():
        if r0 is not None:
            continue
        cfg = _ref_visual_cfg(ref_registry, W, H, n=4)
        if fx is not None:
            cfg.scene.camera.spawn.focal_length = fx
        with pytest.raises(wl.WlError, match="bad camera geometry"):
            env_from_reference_cfg(cfg, device=DEV)
    env = env_from_reference_cfg(_ref_visual_cfg(ref_registry, 124, 49, n=4), device=DEV)      # the control: accepted
    assert env.sim.obs_dim == 4100


@pytest.mark.gpu
def test_policy_act_drives_the_widest_row_it_takes():
    """120 x 34 kept pixels: obs_dim 4088, the widest row wl_policy_act takes (WL_WIDE_MAX_OBS = 4096), against the oracle
    as test_policy_wide_gpu drives the task's 3208."""
    ev._need_gpu()
    import test_policy_wide_gpu as pw
    spec = _spec("120x34", 64, "aug", seed=9)
    assert spec.obs_dim == 4088
    spec.cfg.max_episode_length = 10
    pw._run(spec, 15)


@pytest.mark.gpu
@pytest.mark.parametrize("geom,obs_dim", [("128x32", 4104), ("124x33", 4100)])
def test_device_policy_refuses_rows_wider_than_it_takes(geom, obs_dim):
    """wl_create takes these cameras, the device policy and PPO kernels do not: each refuses with its obs_dim message and
    writes none of its outputs.  The env itself still steps with the oracle."""
    ev._need_gpu()
    import wheeledlab_b200 as wl
    from test_policy_wide_gpu import relu_policy
    from wheeledlab_b200._lib import WlPpoBatch, WlPpoParams, lib
    from wheeledlab_b200.learner import FusedPPO
    from wheeledlab_b200.policy import actor_mean, policy_act
    n = 64
    spec = _spec(geom, n, "aug", seed=9, traversability=_map(9))
    sim, orc = ev._pair(spec)
    assert sim.obs_dim == obs_dim
    obs = sim.observe(0, 0)
    blob = relu_policy(obs_dim)
    sent = lambda *s: _sentinel(int(np.prod(s)), 1).reshape(s)
    untouched = lambda *ts: all(bool((t.view(torch.int32) == int(SENTINEL.view(np.int32))).all()) for t in ts)
    act, mean, lp, val = sent(n, 2), sent(n, 2), sent(n), sent(n)
    with pytest.raises(wl.WlError, match=r"wl_policy_act: obs_dim must be in 1\.\.4096"):
        policy_act(sim, obs, blob, act, mean, lp, val, 0)
    out = sent(n, 2)
    with pytest.raises(wl.WlError, match=r"wl_actor_mean: obs_dim must be in 1\.\.4096"):
        actor_mean(blob, obs_dim, obs, "relu", out)
    torch.cuda.synchronize()
    assert untouched(act, mean, lp, val, out), "a refused policy call wrote its outputs"
    # PPO: a [2, n] slab of these rows
    B = 2 * n
    rows = (obs.repeat(2, 1), sent(B, 2), sent(B), sent(B), sent(B, 2), sent(B), sent(B))
    perm = torch.randperm(B, device=DEV)
    batch = WlPpoBatch(*[x.data_ptr() for x in rows + (perm,)])
    b0 = blob.clone()
    m, v, state, ws = sent(blob.numel()), sent(blob.numel()), sent(int(lib.wl_ppo_state_floats())), sent(1 << 18)
    p = WlPpoParams(obs_dim, B, 5, 4, 0.2, 1.0, 0.005, 1.0, 0.01, 1, 1, 0)
    assert lib.wl_ppo_update_wide(C.byref(p), C.byref(batch), C.c_void_p(blob.data_ptr()), C.c_void_p(m.data_ptr()),
                                  C.c_void_p(v.data_ptr()), C.c_void_p(state.data_ptr()), C.c_void_p(ws.data_ptr()),
                                  4 * ws.numel(), None) == -3
    assert "wl_ppo_update_wide: obs_dim > 4096" in lib.wl_last_error().decode()
    assert lib.wl_ppo_wide_workspace_bytes(obs_dim, B, 4) == 0
    slab = type("Slab", (), dict(zip(("obs_in", "actions", "values", "log_prob", "mean"), rows[:5])))
    with pytest.raises(wl.WlError, match="obs_dim > 4096"):
        FusedPPO(blob, obs_dim, activation="relu").update(slab, rows[5].view(2, n), rows[6].view(2, n), perm)
    torch.cuda.synchronize()
    assert torch.equal(blob.view(torch.int32), b0.view(torch.int32)) and untouched(m, v, state, ws, *rows[1:]), \
        "the refused PPO update wrote its outputs"
    ev._traj(spec, sim, orc, 6, what=f"{geom} after the refusals")
    ev._check_end(sim, orc, geom)


@pytest.mark.gpu
@pytest.mark.parametrize("geom", list(GEOMETRIES))
def test_rollout_refuses_camera_handles(geom):
    ev._need_gpu()
    import wheeledlab_b200 as wl
    from wheeledlab_b200.distributed import RolloutSlab
    for mode in ("raw", "aug"):
        spec = _spec(geom, 4, mode)
        sim = wl.WheeledSim(spec, DEV); sim.startup(); sim.reset(None, 0)
        with pytest.raises(wl.WlError, match="the camera term is a second kernel"):
            sim.rollout(4, 0, RolloutSlab(4, 4, spec.obs_dim, 2, DEV), torch.empty((4, 16), device=DEV))


# ---- 4. the oracle away from 80 x 40 and the fp64 restatements (CPU) ---------------------------------------------------
@pytest.fixture(scope="module")
def ref_registry():
    if str(ROOT / "shims") not in sys.path:
        sys.path.insert(0, str(ROOT / "shims"))
    import recorded_cfgs
    return recorded_cfgs.load()


def _ref_visual_cfg(registry, W, H, n):
    cfg = registry["Isaac-MushrVisualRL-v0"]["cfgs"]["env_cfg_entry_point"]()
    cfg.scene.num_envs = n
    cfg.scene.camera.width, cfg.scene.camera.height = W, H
    return cfg


def test_compat_lowers_a_camera_as_the_helper_sets_it(ref_registry):
    """The recorded Isaac-MushrVisualRL-v0 cfg with its camera resized lowers to the same wl_config, byte for byte, as
    cam_spec on the task (the recorded traversability map's count aside, as in test_compat_cpu)."""
    from wheeledlab_b200.compat import spec_from_reference_cfg
    ref_map = np.load(ROOT / "tests" / "golden" / "cfg_blobs" / "visual_ref_map.npz")["map"]
    blob = lambda c: C.string_at(C.addressof(c), C.sizeof(c))
    for name, (W, H, r0) in GEOMETRIES.items():
        if r0 is not None:
            continue
        got = spec_from_reference_cfg(_ref_visual_cfg(ref_registry, W, H, n=64))
        got.cfg.vis_n_trav = int(ref_map.sum())
        exp = cam_spec(W, H, n=64, camera="aug", seed=42, traversability=ref_map)
        assert blob(got.cfg) == blob(exp.cfg), name
        assert got.obs_dim == exp.obs_dim == 8 + W * (H - H // 3), name


@pytest.mark.parametrize("geom", list(GEOMETRIES))
def test_oracle_render_matches_fp64(geom):
    """The oracle's camera_render at the placed poses against _render64, under the same rule as the kernel."""
    trav = _map(5)
    spec = _spec(geom, len(POSES), "raw", seed=5, traversability=trav)
    orc = O.Oracle(spec.cfg, heightfield=spec.heightfield)
    orc.startup(); orc.reset(None, 0)
    st = _posed(orc.export_state())
    orc.import_state(st)
    W, H, r0 = _geometry(geom)
    got = np.stack([orc.camera_render(i) for i in range(len(POSES))]).reshape(-1, H - r0, W).astype(bool)
    _check_render(spec.cfg, st, trav, got, f"{geom}, oracle")


@pytest.mark.parametrize("geom", list(GEOMETRIES))
def test_oracle_post_processing_matches_fp64(geom):
    W, H, r0 = _geometry(geom)
    white = _masks(W, H - r0, seed=W * 97 + H)
    small = np.ones((8, 8), bool)
    raw = _spec(geom, 1, "raw", traversability=small)
    assert np.abs(O.camera_post(raw.cfg, white, None) - _post64(W, H - r0, white, None)).max() <= 1e-6
    aug = _spec(geom, 1, "aug", traversability=small)
    for j, a in enumerate(AUGS):
        exp = _post64(W, H - r0, white, a)
        for kind in ("f32", "f64"):
            err = np.abs(O.camera_post(aug.cfg, white, a, kind=kind) - exp).max()
            assert err <= 2e-6, f"{geom} parameters {j} ({kind} oracle): max |oracle - fp64| = {err:.3g}"


def test_fp64_post_processing_reproduces_torchvision():
    """_post64 against the reference's own functions (torchvision) at 80 x 40: tests/golden/camera_post.npz."""
    d = np.load(ROOT / "tests" / "golden" / "camera_post.npz")
    white = d["white"]
    assert np.abs(_post64(80, 40, white, None) - d["raw"]).max() <= 1e-6
    for k, a in enumerate(d["aug"]):
        err = np.abs(_post64(80, 40, white, a) - d["out"][k]).max()
        assert err <= 2e-6, (k, err)
