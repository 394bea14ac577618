"""Device event terms (DESIGN 6p) without a GPU: the compat lowering of the reference's own Elevation and Visual cfgs with
IsaacLab's push added in each mode, the refusals by name, the C-ABI's argument checks, and the twin against a numpy
restatement of push_by_setting_velocity on top of the interval timers."""
import ctypes as C
import sys
import types
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(Path(__file__).resolve().parent))

WL_EINVAL = -1
IDS = ["Isaac-MushrElevationRL-v0", "Isaac-MushrVisualRL-v0"]
VR = {"x": (-0.5, 0.5), "yaw": (-1.0, 1.0), "z": (0.0, 0.25)}
RANGES = [(-0.5, 0.5), (0.0, 0.0), (0.0, 0.25), (0.0, 0.0), (0.0, 0.0), (-1.0, 1.0)]


@pytest.fixture(scope="module")
def ref_registry():
    if str(ROOT / "shims") not in sys.path:
        sys.path.insert(0, str(ROOT / "shims"))
    import recorded_cfgs
    return recorded_cfgs.load()


def _push():
    from isaaclab.envs import mdp
    return mdp.push_by_setting_velocity


def _cfg(reg, gid, n=8, **events):
    from isaaclab.managers import EventTermCfg
    c = reg[gid]["cfgs"]["env_cfg_entry_point"]()
    c.scene.num_envs = n
    for name, kw in events.items():
        setattr(c.events, name, EventTermCfg(**kw))
        if hasattr(c.events, "_cfg_fields") and name not in c.events._cfg_fields:
            c.events._cfg_fields = list(c.events._cfg_fields) + [name]
    return c


def _blob(c):
    return C.string_at(C.addressof(c), C.sizeof(c))


def _push_kw(mode, **extra):
    kw = dict(func=_push(), mode=mode, params={"velocity_range": dict(VR)})
    if mode == "interval":
        kw["interval_range_s"] = (1.0, 3.0)
    kw.update(extra)
    return kw


@pytest.mark.parametrize("gid", IDS)
@pytest.mark.parametrize("mode", ["reset", "interval"])
def test_a_push_lowers_to_a_device_event_term(ref_registry, gid, mode):
    from wheeledlab_b200 import device_events as dev
    from wheeledlab_b200.compat import spec_from_reference_cfg
    base = spec_from_reference_cfg(_cfg(ref_registry, gid), device_terms=True)
    spec = spec_from_reference_cfg(_cfg(ref_registry, gid, push=_push_kw(mode)), device_terms=True)
    assert spec.device_events == [("push", _push(), mode, {"velocity_range": VR}, (1.0, 3.0) if mode == "interval" else None)]
    assert dev.velocity_ranges("push", spec.device_events[0][3]) == RANGES
    assert _blob(spec.cfg) == _blob(base.cfg), "a device event changes nothing in the config"
    assert spec.python_event_terms == [] and spec.device_terms == base.device_terms and spec.reset_events == base.reset_events
    # without the flag every path is as before: refused, or a host-side event term with allow_python_terms
    with pytest.raises(NotImplementedError, match="event term push -> push_by_setting_velocity"):
        spec_from_reference_cfg(_cfg(ref_registry, gid, push=_push_kw(mode)))
    py = spec_from_reference_cfg(_cfg(ref_registry, gid, push=_push_kw(mode)), allow_python_terms=True)
    assert py.device_events == [] and [e[0] for e in py.python_event_terms] == ["push"]


def test_the_drift_family_keeps_its_built_in_push_slots(ref_registry):
    from wheeledlab_b200.compat import spec_from_reference_cfg
    for gid in ("Isaac-MushrDriftRL-v0", "Isaac-F1TenthDriftRL-v0"):
        a = spec_from_reference_cfg(_cfg(ref_registry, gid))
        b = spec_from_reference_cfg(_cfg(ref_registry, gid), device_terms=True)
        assert b.device_events == [] and _blob(a.cfg) == _blob(b.cfg), gid


def test_the_committed_cfg_blobs_still_reproduce(ref_registry):
    from wheeledlab_b200.compat import spec_from_reference_cfg
    blobs = ROOT / "tests" / "golden" / "cfg_blobs"
    for gid in ("Isaac-MushrDriftRL-v0", "Isaac-F1TenthDriftRL-v0", "Isaac-MushrElevationRL-v0"):
        for flag in (False, True):
            spec = spec_from_reference_cfg(_cfg(ref_registry, gid, n=4096), device_terms=flag)
            assert spec.device_events == []
            assert _blob(spec.cfg) == (blobs / f"{gid}.ref.bin").read_bytes(), (gid, flag)


@pytest.mark.parametrize("kw,exc,match", [
    (dict(mode="startup"), NotImplementedError, "event term bad: mode 'startup' \\(device event terms run in 'reset' and 'interval'"),
    (dict(mode="prestartup"), NotImplementedError, "event term bad: mode 'prestartup'"),
    (dict(mode="interval", is_global_time=True), NotImplementedError, "event term bad: is_global_time=True"),
    (dict(mode="reset", min_step_count_between_reset=5), NotImplementedError, "event term bad: min_step_count_between_reset 5"),
    (dict(mode="interval", interval_range_s=(2.0, 1.0)), ValueError, "event term bad: interval_range_s"),
    (dict(mode="interval", interval_range_s=(-1.0, 1.0)), ValueError, "event term bad: interval_range_s"),
    (dict(mode="reset", params={"velocity_range": {"x": (1.0, -1.0)}}), ValueError, "event term bad: velocity_range\\['x'\\]"),
    (dict(mode="reset", params={"velocity_range": {"x": (0.0, float("inf"))}}), ValueError, "event term bad: velocity_range\\['x'\\]"),
    (dict(mode="reset", params={"velocity_range": {"w": (0.0, 1.0)}}), ValueError, "event term bad: velocity_range keys \\['w'\\]"),
    (dict(mode="reset", params={"velocity_range": {}, "scale": 2.0}), TypeError, "event term bad: .*unexpected parameters \\['scale'\\]"),
    (dict(mode="reset", params={}), TypeError, "event term bad: .*missing parameter 'velocity_range'"),
])
def test_refusals_by_name(ref_registry, kw, exc, match):
    from wheeledlab_b200.compat import spec_from_reference_cfg
    for gid in IDS:
        with pytest.raises(exc, match=match):
            spec_from_reference_cfg(_cfg(ref_registry, gid, bad=_push_kw(**kw)), device_terms=True)


def test_a_ninth_device_event_is_refused(ref_registry):
    from wheeledlab_b200.compat import spec_from_reference_cfg
    ev = {f"push{k}": _push_kw("interval" if k % 2 else "reset") for k in range(9)}
    with pytest.raises(NotImplementedError, match="event term push8: more than 8 device event terms"):
        spec_from_reference_cfg(_cfg(ref_registry, IDS[0], **ev), device_terms=True)
    ev.pop("push8")
    spec = spec_from_reference_cfg(_cfg(ref_registry, IDS[0], **ev), device_terms=True)
    assert [e[0] for e in spec.device_events] == [f"push{k}" for k in range(8)]


def _fake_env(**kw):
    base = dict(_py_rewards=[], _py_terms=[], _py_events=[], _dev_terms=[], _dev_events=[], _critic_terms=[])
    base.update(kw)
    env = types.SimpleNamespace(**base)
    from wheeledlab_b200.env import ManagerBasedRLEnv
    env._refuse_mixing = lambda device=False: ManagerBasedRLEnv._refuse_mixing(env, device)
    return env


def test_the_env_refuses_by_name_before_any_device_work():
    """add_device_event_term's refusals: a function outside the library, startup mode, Python terms or a critic group on
    the env; and a Python event term on an env with device events."""
    from wheeledlab_b200.env import ManagerBasedRLEnv
    add = ManagerBasedRLEnv.add_device_event_term
    vr = {"velocity_range": dict(VR)}

    def my_kick(env, env_ids, speed=1.0):
        pass

    with pytest.raises(NotImplementedError, match="event term kick: .*my_kick is not in the device event library"):
        add(_fake_env(), "kick", my_kick, "reset", params={"speed": 1.0})
    with pytest.raises(NotImplementedError, match="event term p: mode 'startup'"):
        add(_fake_env(), "p", _push(), "startup", params=vr)
    with pytest.raises(NotImplementedError, match="not both"):
        add(_fake_env(_py_events=[types.SimpleNamespace(name="e")]), "p", _push(), "reset", params=vr)
    with pytest.raises(NotImplementedError, match="not both"):
        add(_fake_env(_py_rewards=[types.SimpleNamespace(name="r")]), "p", _push(), "reset", params=vr)
    with pytest.raises(NotImplementedError, match="a critic observation group together with device terms is not implemented"):
        add(_fake_env(_critic_terms=["base_mass"]), "p", _push(), "interval", (1.0, 2.0), vr)
    with pytest.raises(NotImplementedError, match="not both"):
        ManagerBasedRLEnv._refuse_mixing(_fake_env(_dev_events=[types.SimpleNamespace(name="p")]))
    with pytest.raises(NotImplementedError, match="step_host"):
        ManagerBasedRLEnv.step_host(_fake_env(_dev_events=[types.SimpleNamespace(name="p")]), None)


def test_library_lookup_is_by_module_and_name():
    from wheeledlab_b200 import device_events as dev
    assert dev.lookup(_push()) is dev.PUSH_BY_SETTING_VELOCITY
    assert list(dev.REGISTRY) == [("isaaclab.envs.mdp", "push_by_setting_velocity")]

    def push_by_setting_velocity(env, env_ids, velocity_range):
        pass
    assert dev.lookup(push_by_setting_velocity) is None                 # same name, another module
    from isaaclab.envs import mdp
    assert dev.lookup(mdp.randomize_rigid_body_mass) is None and dev.lookup(lambda env, ids: None) is None


def test_abi_argument_errors_without_a_device():
    import wheeledlab_b200 as wl
    from wheeledlab_b200._lib import WlDeviceEventDesc
    lib = wl.lib
    assert C.sizeof(WlDeviceEventDesc) == 60
    table = (WlDeviceEventDesc * 1)()
    table[0].mode = 1
    buf = (C.c_uint8 * 16)()
    assert lib.wl_set_device_events(None, table, 1) == WL_EINVAL
    assert b"wl_set_device_events" in lib.wl_last_error()
    assert lib.wl_device_events(None, buf, buf, 0, None) == WL_EINVAL
    assert b"wl_device_events" in lib.wl_last_error()


# ---- the twin against a numpy restatement of push_by_setting_velocity on the interval timers ---------------------------------
def _u(r):
    return (r >> np.uint32(8)).astype(np.float32) * np.float32(5.9604644775390625e-08)


def _numpy_events(seed, off, n, table, dt, dones, vel):
    """Timers as EventManager's (test_event_terms_cpu restates them); then, per term in order, where it fires:
    root_vel_w += rand * (hi - lo) + lo per component (sample_uniform)."""
    from oracle_lib import philox
    from test_event_terms_cpu import _numpy_timers
    timers = [r for mode, r, _ in table if mode == "interval"]
    tl = _numpy_timers(seed, off, n, timers, dt, dones) if timers else None
    out = []
    for t, done in enumerate(dones):
        j = 0
        for k, (mode, _, ranges) in enumerate(table):
            if mode == "interval":
                f = tl[t][0][j] != 0
                j += 1
            else:
                f = done != 0
            a, b = philox(seed, off, t, 15, k, n), philox(seed, off, t, 15, 8 + k, n)
            r = np.concatenate([a, b[:, :2]], axis=1)
            lo = np.asarray([x[0] for x in ranges], np.float32)
            hi = np.asarray([x[1] for x in ranges], np.float32)
            vel = np.where(f[:, None], vel + (_u(r) * (hi - lo) + lo), vel)
        out.append(vel.copy())
    return out


def test_twin_equals_the_numpy_restatement():
    import device_events_oracle as deo
    seed, n, dt = 99, 41, np.float32(0.1)
    rng = np.random.default_rng(2)
    table = [("interval", (0.2, 0.6), RANGES), ("reset", None, [(-1.0, 1.0)] * 6), ("interval", (0.0, 0.0), [(0.0, 0.0)] * 6),
             ("interval", (0.05, 0.3), [(0.1, 0.2), (-0.3, -0.1), (0.0, 0.0), (0.5, 0.5), (-2.0, 2.0), (0.0, 1.0)])]
    dones = [(rng.random(n) < p).astype(np.uint8) for p in [0.0, 1.0] + [0.1] * 28]
    for off in (0, 500):
        for tb in (table[:1], table[1:2], table):
            vel0 = rng.standard_normal((n, 6)).astype(np.float32)
            want = _numpy_events(seed, off, n, tb, dt, dones, vel0.copy())
            tl, vel = deo.init(seed, off, n, tb), vel0.copy()
            for t, done in enumerate(dones):
                deo.step(seed, off, tb, dt, done, tl, vel, t)
                assert np.array_equal(vel.view(np.uint32), want[t].view(np.uint32)), (off, len(tb), t)
            assert not np.array_equal(vel, vel0)


def test_twin_does_not_depend_on_sharding():
    import device_events_oracle as deo
    seed, n, dt = 3, 64, np.float32(0.1)
    table = [("interval", (0.1, 0.4), RANGES), ("reset", None, [(-0.1, 0.3)] * 6)]
    rng = np.random.default_rng(4)
    vel = rng.standard_normal((n, 6)).astype(np.float32)
    halves = [vel[:32].copy(), vel[32:].copy()]
    tl, th = deo.init(seed, 0, n, table), [deo.init(seed, 0, 32, table), deo.init(seed, 32, 32, table)]
    for t in range(30):
        done = (rng.random(n) < 0.1).astype(np.uint8)
        deo.step(seed, 0, table, dt, done, tl, vel, t)
        for h in (0, 1):
            deo.step(seed, 32 * h, table, dt, done[32 * h:32 * h + 32], th[h], halves[h], t)
        assert np.array_equal(vel, np.concatenate(halves)) and np.array_equal(tl, np.concatenate(th, axis=1))
