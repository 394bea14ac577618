"""ctypes wrapper of the CPU oracle (oracle/wl_oracle.c).  TEST INFRASTRUCTURE ONLY."""
from __future__ import annotations

import atexit
import ctypes as C
import os
import shutil
import subprocess
import tempfile
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
ODIR = ROOT / "oracle"


def _ensure_built(native=False):
    in_tree = [ODIR / "libwl_oracle.so", ODIR / "libwl_oracle_f64.so"]
    if not (all(p.exists() for p in in_tree) and not os.access(ODIR, os.W_OK)):     # a read-only tree is used as built
        subprocess.run(["make", "-C", str(ODIR), *(p.name for p in in_tree)], check=True, stdout=subprocess.DEVNULL)
    if not native:
        return None
    # the host-tuned build is made for the host that runs it, outside the (possibly read-only) source tree
    out = Path(tempfile.mkdtemp(prefix="wl_oracle_native_"))
    atexit.register(shutil.rmtree, out, True)
    subprocess.run(["make", "-C", str(ODIR), f"NATIVE_DIR={out}", str(out / "libwl_oracle_native.so")], check=True, stdout=subprocess.DEVNULL)
    return out


def _load(path):
    lib = C.CDLL(str(path))
    vp, i32, i64, u32, u64 = C.c_void_p, C.c_int32, C.c_int64, C.c_uint32, C.c_uint64
    lib.wlo_create.restype = vp
    lib.wlo_create.argtypes = [vp, vp]
    lib.wlo_destroy.argtypes = [vp]
    lib.wlo_startup.argtypes = [vp]
    lib.wlo_reset.argtypes = [vp, vp, i32, i64]
    lib.wlo_step.argtypes = [vp, vp, vp, vp, vp, vp, i64, i32]
    lib.wlo_observe.argtypes = [vp, vp, i64, i32]
    lib.wlo_curriculum.argtypes = [vp, i32, vp, vp, u32]
    lib.wlo_synth_actions.argtypes = [vp, vp, i64, i32]
    lib.wlo_export_state.argtypes = [vp, vp]
    lib.wlo_import_state.argtypes = [vp, vp]
    lib.wlo_get_weights.argtypes = [vp, vp]
    lib.wlo_set_weights.argtypes = [vp, vp]
    lib.wlo_get_log.argtypes = [vp, vp]
    lib.wlo_any_reset_last.argtypes = [vp]
    lib.wlo_detmath.argtypes = [i32, vp, vp, vp, i32]
    lib.wlo_philox.argtypes = [u64, u32, u32, u32, u32, vp, i32]
    lib.wlo_action_map.argtypes = [vp, vp, vp, vp, i32]
    lib.wlo_drift_terms.argtypes = [vp, vp, vp, vp, vp, vp, i32]
    lib.wlo_euler_xyz.argtypes = [vp, vp, i32]
    lib.wlo_drift_reset_pose.argtypes = [vp, vp, vp, vp, vp, i32]
    lib.wlo_elev_terms.argtypes = [vp, vp, vp, vp, vp, vp, vp, vp, vp, i32]
    lib.wlo_dc_motor.argtypes = [vp, C.c_float, C.c_float, vp, vp, vp, i32]
    lib.wlo_camera.argtypes = [vp, vp, i64, vp]
    lib.wlo_camera_post.argtypes = [vp, vp, vp, vp, i32]
    lib.wlo_camera_render.argtypes = [vp, i32, vp]
    lib.wlo_derive_suspension.argtypes = [vp, vp, vp]
    lib.wlo_set_device_terms.argtypes = [vp, vp, i32]
    lib.wlo_step_terms.argtypes = [vp, vp, vp, vp, vp, vp, i64, i32]
    lib.wlo_get_device_terms.argtypes = [vp, vp, vp, vp, vp]
    lib.wlo_device_terms.argtypes = [vp, vp, vp, i32, vp, vp, i64, vp, vp, vp, vp, vp, vp]
    lib.wlo_set_reset_events.argtypes = [vp, u32]
    lib.wlo_event_timers_init.argtypes = [u64, i32, i32, i32, vp, vp]
    lib.wlo_event_timers.argtypes = [u64, i32, i32, i32, vp, C.c_float, vp, vp, vp, i64]
    lib.wlo_device_events.argtypes = [u64, i32, i32, i32, vp, vp, vp, i32, vp, C.c_float, vp, vp, vp, i64]
    lib.wlo_policy_observe.argtypes = [u64, i32, i32, vp, i32, vp, vp, vp, vp, vp, vp, vp, vp, vp, i32, u32, i32, vp]
    lib.wlo_policy_library.argtypes = [vp, i32, vp]
    lib.wlo_policy_obs_draw.argtypes = [u64, u32, u32, i32, i32, i32]
    lib.wlo_policy_obs_draw.restype = C.c_float
    lib.wlo_config_describe.restype = C.c_char_p
    return lib


_libs = {}


def get_lib(kind="f32"):
    if kind not in _libs:
        ndir = _ensure_built(native=(kind == "native"))
        _libs[kind] = _load(ndir / "libwl_oracle_native.so" if kind == "native" else ODIR / {"f32": "libwl_oracle.so", "f64": "libwl_oracle_f64.so"}[kind])
    return _libs[kind]


def _p(a):
    return C.c_void_p(a.ctypes.data) if a is not None else None


NUM_GROUPS = 16

_CFG_CLS = None


def config_struct():
    """ctypes mirror of wl_config built from the ORACLE's own field list (wlo_config_describe), so that the reference arm of
    bench.py can drive the oracle from a committed config blob without importing the product package."""
    global _CFG_CLS
    if _CFG_CLS is None:
        tags = {"i32": C.c_int32, "u64": C.c_uint64, "f32": C.c_float}
        fields, size = [], None
        for item in get_lib().wlo_config_describe().decode().split(";"):
            if not item:
                continue
            parts = item.split(":")
            if parts[0] == "sizeof":
                size = int(parts[1]); continue
            ct = tags[parts[1]]
            fields.append((parts[0], ct if int(parts[2]) == 1 else ct * int(parts[2])))
        _CFG_CLS = type("WloConfig", (C.Structure,), {"_fields_": fields})
        assert size is None or C.sizeof(_CFG_CLS) == size
    return _CFG_CLS


def cfg_from_blob(path, **overrides):
    """wl_config from a binary blob (python -m wheeledlab_b200.dump_config / tests/golden/cfg_blobs) + field overrides."""
    cls = config_struct()
    raw = Path(path).read_bytes()
    assert len(raw) == C.sizeof(cls), f"{path}: {len(raw)} bytes, wl_config is {C.sizeof(cls)} (stale blob? regenerate)"
    cfg = cls.from_buffer_copy(raw)
    for k, v in overrides.items():
        setattr(cfg, k, v)
    return cfg


class TermDesc(C.Structure):
    """wl_term_desc"""
    _fields_ = [("kind", C.c_int32), ("role", C.c_int32), ("weight", C.c_double), ("params", C.c_double * 4)]


MAX_DEVICE_TERMS = 8


def term_table(terms):
    """A wl_term_desc array from (kind, role, weight, params[<= 4]) rows."""
    arr = (TermDesc * max(1, len(terms)))()
    for k, (kind, role, weight, params) in enumerate(terms):
        p = list(params) + [0.0] * (4 - len(params))
        arr[k] = TermDesc(int(kind), int(role), float(weight), (C.c_double * 4)(*p))
    return arr


def device_terms(cfg, terms, state, done, t, vis_map=None, prev=None, sums=None, rew=None, kind="f32"):
    """wlo_device_terms: the term kernel on placed states (state [16, N, 4] float32, done [N]).  Returns a dict of rew [N],
    fired [N], vals [N, 8], term_log [8], prev [N] and sums [8, N] (float64; fp32 values in the fp32 build)."""
    n = int(cfg.num_envs)
    st = np.ascontiguousarray(state, np.float32)
    assert st.shape == (NUM_GROUPS, n, 4)
    dn = np.ascontiguousarray(done, np.uint8)
    out = {"prev": np.full(n, np.nan) if prev is None else np.array(prev, np.float64),
           "sums": np.zeros((MAX_DEVICE_TERMS, n)) if sums is None else np.array(sums, np.float64),
           "rew": np.zeros(n) if rew is None else np.array(rew, np.float64),
           "fired": np.zeros(n, np.uint8), "vals": np.zeros((n, MAX_DEVICE_TERMS)), "term_log": np.zeros(MAX_DEVICE_TERMS)}
    m = None if vis_map is None else np.ascontiguousarray(vis_map, np.uint8)
    tt = term_table(terms)
    rc = get_lib(kind).wlo_device_terms(C.byref(cfg), _p(m), tt, len(terms), _p(st), _p(dn), int(t), _p(out["prev"]),
                                        _p(out["sums"]), _p(out["rew"]), _p(out["fired"]), _p(out["vals"]), _p(out["term_log"]))
    assert rc == 0, rc
    return out


def event_timers_init(seed, env_id_offset, n, ranges) -> np.ndarray:
    """wlo_event_timers_init: the interval timers [n_terms, N] f32 of (lo, hi) ranges as wl_set_event_timers draws them."""
    lo_hi = np.ascontiguousarray(ranges, dtype=np.float32).reshape(-1)
    tl = np.zeros((len(ranges), n), dtype=np.float32)
    get_lib().wlo_event_timers_init(seed, env_id_offset, n, len(ranges), _p(lo_hi), _p(tl))
    return tl


def event_timers_step(seed, env_id_offset, ranges, step_dt, done, time_left, step_counter):
    """wlo_event_timers: one step in place on time_left; returns fired [n_terms, N] u8."""
    lo_hi = np.ascontiguousarray(ranges, dtype=np.float32).reshape(-1)
    n = time_left.shape[1]
    done = np.ascontiguousarray(done, dtype=np.uint8)
    fired = np.zeros(time_left.shape, dtype=np.uint8)
    get_lib().wlo_event_timers(seed, env_id_offset, n, len(ranges), _p(lo_hi), np.float32(step_dt), _p(done), _p(time_left),
                               _p(fired), step_counter)
    return fired


# A device event table is a list of (mode, interval_range_s or None, six (lo, hi) velocity ranges), as
# WheeledSim.set_device_events takes it.
def _timer_ranges(table):
    return [tuple(r) for mode, r, _ in table if mode == "interval"]


def device_events_init(seed, env_id_offset, n, table) -> np.ndarray:
    """The interval terms' timers as wl_set_device_events draws them: [n_interval_terms, N] f32."""
    ranges = _timer_ranges(table)
    return event_timers_init(seed, env_id_offset, n, ranges) if ranges else np.zeros((0, n), np.float32)


def device_events_step(seed, env_id_offset, table, step_dt, done, time_left, vel, step_counter):
    """wlo_device_events: one step of every term, in place on time_left [n_interval_terms, N] f32 and vel [N, 6] f32 (x, y, z,
    roll, pitch, yaw)."""
    n = vel.shape[0]
    slot, j = [], 0
    for mode, _, _ in table:
        slot.append(j if mode == "interval" else -1)
        j += mode == "interval"
    slot = np.asarray(slot or [0], dtype=np.int32)
    lo = np.ascontiguousarray([[r[0] for r in rr] for _, _, rr in table] or [[0.0] * 6], dtype=np.float32)
    hi = np.ascontiguousarray([[r[1] for r in rr] for _, _, rr in table] or [[0.0] * 6], dtype=np.float32)
    tlh = np.ascontiguousarray(_timer_ranges(table) or [(0.0, 0.0)], dtype=np.float32).reshape(-1)
    done = np.ascontiguousarray(done, dtype=np.uint8)
    assert vel.dtype == np.float32 and vel.flags.c_contiguous and time_left.dtype == np.float32 and time_left.flags.c_contiguous
    get_lib().wlo_device_events(seed, env_id_offset, n, len(table), _p(slot), _p(lo), _p(hi), j, _p(tlh), np.float32(step_dt), _p(done),
                                _p(time_left), _p(vel), step_counter)


# A policy observation table is a list of (library name, noise, clip, scale) as WheeledSim.set_policy_terms takes it; the state
# is the device state's groups, float32 [NUM_GROUPS, N, 4] (sim.groups).
# First library float and width of each term (the row the kernel forms per env: the critic library, then gravity).
LIBRARY = {"root_pos_w": (0, 3), "root_euler_xyz": (3, 3), "base_lin_vel": (6, 3), "base_ang_vel": (9, 3), "last_action": (12, 2),
           "joint_vel": (14, 4), "joint_pos": (18, 2), "wheel_friction": (20, 4), "base_mass": (24, 1), "motor_damping": (25, 4),
           "projected_gravity": (29, 3)}
NOISE = {None: 0, "gaussian": 1, "uniform": 2}


def policy_columns(table) -> dict:
    """Per output column: src, noise kind, (na, nb) = (mean, std) or (n_min, n_max - n_min) with the span formed in double,
    clip flag and bounds, scale flag and value -- each parameter rounded to fp32."""
    cols = {k: [] for k in ("src", "noise", "na", "nb", "has_clip", "lo", "hi", "has_scale", "scale")}
    for name, noise, clip, scale in table:
        first, width = LIBRARY[name]
        sc = None if scale is None else ((float(scale),) if isinstance(scale, (int, float)) else tuple(float(s) for s in scale))
        for k in range(width):
            cols["src"].append(first + k)
            cols["noise"].append(NOISE[None if noise is None else noise[0]])
            a, b = (0.0, 0.0) if noise is None else (float(noise[1]), float(noise[2]))
            cols["na"].append(a)
            cols["nb"].append(b - a if noise is not None and noise[0] == "uniform" else b)
            cols["has_clip"].append(clip is not None)
            cols["lo"].append(0.0 if clip is None else float(clip[0]))
            cols["hi"].append(0.0 if clip is None else float(clip[1]))
            cols["has_scale"].append(sc is not None)
            cols["scale"].append(1.0 if sc is None else sc[0 if len(sc) == 1 else k])
    out = {}
    for k, v in cols.items():
        dt = np.uint8 if k in ("src", "noise", "has_clip", "has_scale") else np.float32
        out[k] = np.ascontiguousarray(np.asarray(v or [0], dtype=np.float64 if dt is np.float32 else np.int64).astype(dt))
    return out


def policy_observe(seed, env_id_offset, st, table, corrupt, t, call_idx=-1) -> np.ndarray:
    """wlo_policy_observe: the policy row [N, Dp] of the state groups st [G, N, 4] for the step at t (call_idx -1) or an
    observe call."""
    st = np.ascontiguousarray(st, dtype=np.float32)
    n = st.shape[1]
    c = policy_columns(table)
    dp = sum(LIBRARY[name][1] for name, *_ in table)
    out = np.zeros((n, max(dp, 1)), dtype=np.float32)
    get_lib().wlo_policy_observe(seed, env_id_offset, n, _p(st), dp, _p(c["src"]), _p(c["noise"]), _p(c["na"]), _p(c["nb"]),
                                 _p(c["has_clip"]), _p(c["lo"]), _p(c["hi"]), _p(c["has_scale"]), _p(c["scale"]), int(bool(corrupt)),
                                 t & 0xFFFFFFFF, call_idx, _p(out))
    return out[:, :dp]


def policy_library(st) -> np.ndarray:
    """wlo_policy_library: [N, 32] library floats of every env."""
    st = np.ascontiguousarray(st, dtype=np.float32)
    out = np.zeros((st.shape[1], 32), dtype=np.float32)
    get_lib().wlo_policy_library(_p(st), st.shape[1], _p(out))
    return out


def policy_draw(seed, gid, t, call_idx, j, kind) -> np.float32:
    """wlo_policy_obs_draw: the noise draw of column j, z (kind "gaussian") or u in [0, 1) (kind "uniform")."""
    return np.float32(get_lib().wlo_policy_obs_draw(seed, gid, t & 0xFFFFFFFF, call_idx, j, NOISE[kind]))


class Oracle:
    """One oracle instance; mirrors the wl_* calls with host (numpy) buffers."""

    def __init__(self, cfg, heightfield=None, kind="f32", threads=1):
        self.lib = get_lib(kind)
        self.cfg = cfg
        self.n = int(cfg.num_envs)
        self.threads = threads
        self.obs_dim = {0: 14, 1: 689, 2: 8}[int(cfg.task)]
        if int(cfg.task) == 2 and int(cfg.vis_cam):
            self.obs_dim += int(cfg.vis_cam_w) * (int(cfg.vis_cam_h) - int(cfg.vis_cam_row0))
        if heightfield is None:
            hf = None
        elif int(cfg.task) == 2:
            hf = np.ascontiguousarray(heightfield)                      # raw aux bytes (visual)
        else:
            hf = np.ascontiguousarray(heightfield, dtype=np.float32)
        self._h = C.c_void_p(self.lib.wlo_create(C.byref(cfg), _p(hf)))

    def __del__(self):
        try:
            self.lib.wlo_destroy(self._h)
        except Exception:
            pass

    def startup(self):
        assert self.lib.wlo_startup(self._h) == 0

    def reset(self, env_ids, step_counter):
        if env_ids is None:
            rc = self.lib.wlo_reset(self._h, None, 0, step_counter)
        else:
            ids = np.ascontiguousarray(env_ids, dtype=np.int64)
            rc = self.lib.wlo_reset(self._h, _p(ids), len(ids), step_counter)
        assert rc == 0

    def step(self, action, step_counter):
        a = np.ascontiguousarray(action, dtype=np.float32)
        obs = np.empty((self.n, self.obs_dim), np.float32)
        rew = np.empty(self.n, np.float32)
        term = np.empty(self.n, np.uint8)
        trunc = np.empty(self.n, np.uint8)
        rc = self.lib.wlo_step(self._h, _p(a), _p(obs), _p(rew), _p(term), _p(trunc), step_counter, self.threads)
        assert rc == 0, rc
        return obs, rew, term, trunc

    def set_device_terms(self, terms):
        """wl_set_device_terms: (kind, role, weight, params) rows; [] clears them."""
        assert self.lib.wlo_set_device_terms(self._h, term_table(terms), len(terms)) == 0

    def set_reset_events(self, mask) -> int:
        """wl_set_reset_events: the WL_RESET_EV_* bits step, step_terms and reset redraw; 0, or WL_EINVAL with the mask left
        as it was."""
        return self.lib.wlo_set_reset_events(self._h, mask)

    def step_terms(self, action, step_counter):
        """wl_step_terms: step() with the device terms; returns (obs, rew, term, trunc, fired [N], term_log [8])."""
        a = np.ascontiguousarray(action, dtype=np.float32)
        obs = np.empty((self.n, self.obs_dim), np.float32)
        rew = np.empty(self.n, np.float32)
        term = np.empty(self.n, np.uint8)
        trunc = np.empty(self.n, np.uint8)
        rc = self.lib.wlo_step_terms(self._h, _p(a), _p(obs), _p(rew), _p(term), _p(trunc), step_counter, self.threads)
        assert rc == 0, rc
        fired = np.empty(self.n, np.uint8)
        tl = np.empty(MAX_DEVICE_TERMS, np.float64)
        assert self.lib.wlo_get_device_terms(self._h, _p(fired), _p(tl), None, None) == 0
        return obs, rew, term, trunc, fired, tl

    def observe(self, step_counter, call_idx=0):
        obs = np.empty((self.n, self.obs_dim), np.float32)
        assert self.lib.wlo_observe(self._h, _p(obs), step_counter, call_idx) == 0
        return obs

    def curriculum(self, slots, increases, fire_mask):
        s = np.asarray(slots, np.int32)
        i = np.asarray(increases, np.float32)
        assert self.lib.wlo_curriculum(self._h, len(s), _p(s), _p(i), fire_mask) == 0

    def synth_actions(self, step_counter, dist=0):
        a = np.empty((self.n, 2), np.float32)
        assert self.lib.wlo_synth_actions(C.byref(self.cfg), _p(a), step_counter, dist) == 0
        return a

    def export_state(self):
        buf = np.zeros((NUM_GROUPS, self.n, 4), np.float32)
        self.lib.wlo_export_state(self._h, _p(buf))
        return buf

    def import_state(self, buf):
        b = np.ascontiguousarray(buf, dtype=np.float32)
        self.lib.wlo_import_state(self._h, _p(b))

    def weights(self):
        w = np.zeros(8, np.float32)
        self.lib.wlo_get_weights(self._h, _p(w))
        return w

    def set_weights(self, w):
        w = np.ascontiguousarray(w, np.float32)
        self.lib.wlo_set_weights(self._h, _p(w))

    def camera(self, step_counter, aug=None):
        """Camera term alone into a fresh [n, obs_dim] buffer (only the camera floats are written)."""
        obs = np.zeros((self.n, self.obs_dim), np.float32)
        a = None if aug is None else np.ascontiguousarray(aug, np.float32)
        assert self.lib.wlo_camera(self._h, _p(obs), step_counter, _p(a)) == 0
        return obs

    def camera_render(self, li):
        npix = self.obs_dim - 8
        out = np.zeros(npix, np.uint8)
        assert self.lib.wlo_camera_render(self._h, li, _p(out)) == 0
        return out

    def suspension(self):
        """Derived suspension joint state of the current state (wl_derive_suspension): (pos [n,4], vel [n,4]), wheel order
        [bl, br, fl, fr]."""
        pos = np.empty((self.n, 4), np.float32)
        vel = np.empty((self.n, 4), np.float32)
        assert self.lib.wlo_derive_suspension(self._h, _p(pos), _p(vel)) == 0
        return pos, vel

    def any_reset(self) -> bool:
        """>= 1 env reset in the most recent step (the log row itself persists over steps without a reset)."""
        return bool(self.lib.wlo_any_reset_last(self._h))

    def log(self):
        out = np.zeros(16, np.float64)
        self.lib.wlo_get_log(self._h, _p(out))
        return out


def detmath(op, x, x2=None, kind="f32"):
    lib = get_lib(kind)
    x = np.ascontiguousarray(x, np.float32)
    x2 = x if x2 is None else np.ascontiguousarray(x2, np.float32)
    out = np.empty_like(x)
    assert lib.wlo_detmath(op, _p(x), _p(x2), _p(out), x.size) == 0
    return out


def dc_motor(cfg, kd, effort_limit, target, omega):
    t = np.ascontiguousarray(target, np.float32); w = np.ascontiguousarray(omega, np.float32)
    out = np.empty_like(t)
    assert get_lib().wlo_dc_motor(C.byref(cfg), kd, effort_limit, _p(t), _p(w), _p(out), t.size) == 0
    return out


def camera_post(cfg, white, aug, kind="f32"):
    """camera_data_rgb_flattened[_aug] on white masks [n, rows*W] with explicit ColorJitter / blur parameters (9 floats)."""
    white = np.ascontiguousarray(white, np.uint8)
    out = np.empty(white.shape, np.float32)
    a = None if aug is None else np.ascontiguousarray(aug, np.float32)
    assert get_lib(kind).wlo_camera_post(C.byref(cfg), _p(white), _p(a), _p(out), white.shape[0]) == 0
    return out


def philox(seed, c0_base, c1, c2, c3, n):
    out = np.empty((n, 4), np.uint32)
    assert get_lib().wlo_philox(seed, c0_base, c1, c2, c3, _p(out), n) == 0
    return out


def action_map(cfg, action):
    a = np.ascontiguousarray(action, np.float32)
    n = a.shape[0]
    wheel = np.empty((n, 4), np.float32)
    steer = np.empty((n, 2), np.float32)
    rc = get_lib().wlo_action_map(C.byref(cfg), _p(a), _p(wheel), _p(steer), n)
    assert rc == 0, rc
    return wheel, steer


def drift_terms(cfg, root, steer, ep_len):
    root = np.ascontiguousarray(root, np.float32)
    steer = np.ascontiguousarray(steer, np.float32)
    ep = np.ascontiguousarray(ep_len, np.int32)
    n = root.shape[0]
    f = np.empty((n, 8), np.float32)
    oob = np.empty(n, np.uint8)
    assert get_lib().wlo_drift_terms(C.byref(cfg), _p(root), _p(steer), _p(ep), _p(f), _p(oob), n) == 0
    return f, oob


def euler_xyz(quat):
    q = np.ascontiguousarray(quat, np.float32)
    out = np.empty((q.shape[0], 3), np.float32)
    assert get_lib().wlo_euler_xyz(_p(q), _p(out), q.shape[0]) == 0
    return out


def drift_reset_pose(cfg, idx, u_xy, u_yaw):
    idx = np.ascontiguousarray(idx, np.int32)
    u_xy = np.ascontiguousarray(u_xy, np.float32)
    u_yaw = np.ascontiguousarray(u_yaw, np.float32)
    pose = np.empty((idx.shape[0], 7), np.float32)
    assert get_lib().wlo_drift_reset_pose(C.byref(cfg), _p(idx), _p(u_xy), _p(u_yaw), _p(pose), idx.shape[0]) == 0
    return pose


def elev_terms(cfg, root, cmdb, omega, action, ep_len):
    root = np.ascontiguousarray(root, np.float32); cmdb = np.ascontiguousarray(cmdb, np.float32)
    omega = np.ascontiguousarray(omega, np.float32); action = np.ascontiguousarray(action, np.float32)
    ep = np.ascontiguousarray(ep_len, np.int32)
    n = root.shape[0]
    f = np.empty((n, 8), np.float32); mask = np.empty(n, np.uint32); prop = np.empty((n, 13), np.float32)
    assert get_lib().wlo_elev_terms(C.byref(cfg), _p(root), _p(cmdb), _p(omega), _p(action), _p(ep), _p(f), _p(mask), _p(prop), n) == 0
    return f, mask, prop
