"""Host-side event terms (DESIGN 6o) without a GPU: the compat lowering of the reference's own cfg objects with a user event
added in each mode, the refusals by name, the C-ABI's argument checks, and the interval timers' CPU twin against a numpy
restatement of IsaacLab's EventManager timers."""
import ctypes as C
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(Path(__file__).resolve().parent))

WL_EINVAL = -1


@pytest.fixture(scope="module")
def ref_registry():
    if str(ROOT / "shims") not in sys.path:
        sys.path.insert(0, str(ROOT / "shims"))
    import recorded_cfgs
    return recorded_cfgs.load()


def my_spawn(env, env_ids, spread=0.5):
    pass


def my_kick(env, env_ids, speed=1.0):
    pass


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


@pytest.mark.parametrize("gid", ["Isaac-MushrDriftRL-v0", "Isaac-MushrElevationRL-v0"])
@pytest.mark.parametrize("mode", ["startup", "reset", "interval"])
def test_a_user_event_lowers_to_a_python_event_term(ref_registry, gid, mode):
    from wheeledlab_b200.compat import spec_from_reference_cfg
    kw = dict(func=my_spawn if mode != "interval" else my_kick, mode=mode, params={"spread": 0.25} if mode != "interval" else {"speed": 2.0})
    if mode == "interval":
        kw["interval_range_s"] = (1.0, 3.0)
    base = spec_from_reference_cfg(_cfg(ref_registry, gid))
    spec = spec_from_reference_cfg(_cfg(ref_registry, gid, my_event=kw), allow_python_terms=True)
    want = ("my_event", kw["func"], mode, kw["params"], (1.0, 3.0) if mode == "interval" else None)
    assert spec.python_event_terms == [want]
    assert _blob(spec.cfg) == _blob(base.cfg), "a Python event changes nothing in the config"
    assert spec.reset_events == base.reset_events and spec.python_reward_terms == [] and spec.python_termination_terms == []
    with pytest.raises(NotImplementedError, match="event term my_event -> my_"):
        spec_from_reference_cfg(_cfg(ref_registry, gid, my_event=kw))


def test_a_cfg_without_user_events_lowers_to_the_committed_blob(ref_registry):
    from wheeledlab_b200.compat import spec_from_reference_cfg
    blobs = ROOT / "tests" / "golden" / "cfg_blobs"
    for gid in ("Isaac-MushrDriftRL-v0", "Isaac-F1TenthDriftRL-v0", "Isaac-MushrElevationRL-v0"):
        spec = spec_from_reference_cfg(_cfg(ref_registry, gid, n=4096), allow_python_terms=True)
        assert spec.python_event_terms == []
        assert _blob(spec.cfg) == (blobs / f"{gid}.ref.bin").read_bytes(), gid


@pytest.mark.parametrize("kw,match", [
    (dict(mode="prestartup"), "event term bad: mode 'prestartup'"),
    (dict(mode="interval", interval_range_s=(1.0, 2.0), is_global_time=True), "event term bad: is_global_time=True"),
    (dict(mode="reset", min_step_count_between_reset=5), "event term bad: min_step_count_between_reset 5"),
    (dict(mode="bogus"), "event term bad: mode 'bogus'"),
])
def test_refusals_by_name(ref_registry, kw, match):
    from wheeledlab_b200.compat import spec_from_reference_cfg
    for gid in ("Isaac-MushrDriftRL-v0", "Isaac-MushrElevationRL-v0"):
        with pytest.raises(NotImplementedError, match=match):
            spec_from_reference_cfg(_cfg(ref_registry, gid, bad=dict(func=my_spawn, **kw)), allow_python_terms=True)


def test_more_than_eight_interval_terms_and_bad_ranges_are_refused(ref_registry):
    from wheeledlab_b200.compat import check_event_term, spec_from_reference_cfg
    ev = {f"kick{k}": dict(func=my_kick, mode="interval", interval_range_s=(1.0, 2.0)) for k in range(9)}
    with pytest.raises(NotImplementedError, match="event term kick8: more than 8 Python interval event terms"):
        spec_from_reference_cfg(_cfg(ref_registry, "Isaac-MushrDriftRL-v0", **ev), allow_python_terms=True)
    ev.pop("kick8")
    spec = spec_from_reference_cfg(_cfg(ref_registry, "Isaac-MushrDriftRL-v0", **ev), allow_python_terms=True)
    assert [e[0] for e in spec.python_event_terms] == [f"kick{k}" for k in range(8)]
    for rng in (None, (2.0, 1.0), (-0.5, 1.0), (0.0, float("inf"))):
        with pytest.raises(ValueError, match="event term x: "):
            check_event_term("x", "interval", rng)


def test_built_in_events_keep_their_refusals(ref_registry):
    """A built-in DR event in interval mode is refused as before, with or without allow_python_terms."""
    from wheeledlab_b200.compat import spec_from_reference_cfg
    for flag in (False, True):
        c = _cfg(ref_registry, "Isaac-MushrDriftRL-v0")
        c.events.change_wheel_friction.mode = "interval"
        with pytest.raises(NotImplementedError, match="event term change_wheel_friction: mode 'interval'"):
            spec_from_reference_cfg(c, allow_python_terms=flag)


def test_abi_argument_errors_without_a_device():
    import wheeledlab_b200 as wl
    lib = wl.lib
    lo_hi = (C.c_float * 2)(0.5, 1.0)
    buf = (C.c_uint8 * 16)()
    assert lib.wl_set_event_timers(None, 1, lo_hi) == WL_EINVAL
    assert b"wl_set_event_timers" in lib.wl_last_error()
    assert lib.wl_event_timers(None, buf, buf, 0, None) == WL_EINVAL
    assert b"wl_event_timers" in lib.wl_last_error()
    assert lib.wl_step_stage_b1(None, buf, None, None, buf, buf, None, 0, None) == WL_EINVAL
    assert b"wl_step_stage_b1" in lib.wl_last_error()
    assert lib.wl_step_stage_b2(None, buf, 0, None) == WL_EINVAL
    assert b"wl_step_stage_b2" in lib.wl_last_error()


# ---- the interval timers' twin against a numpy restatement of EventManager's timers ----------------------------------------
def _interval(r, lo, hi):
    u = (r >> np.uint32(8)).astype(np.float32) * np.float32(5.9604644775390625e-08)
    return u * (np.float32(hi) - np.float32(lo)) + np.float32(lo)      # (the bounds are fp32 in the handle's table)


def _numpy_timers(seed, off, n, ranges, dt, dones):
    """time_left[k] ~ U[lo, hi) at construction; each step: redraw where done, -= dt, fire where < 1e-6 and redraw there."""
    from oracle_lib import philox
    tl = np.stack([_interval(philox(seed, off, 0, 14, k, n)[:, 0], *ranges[k]) for k in range(len(ranges))])
    out = []
    for t, done in enumerate(dones):
        fired = np.zeros(tl.shape, np.uint8)
        for k, (lo, hi) in enumerate(ranges):
            r = philox(seed, off, t, 13, k, n)
            x = np.where(done != 0, _interval(r[:, 0], lo, hi), tl[k])
            x = x - np.float32(dt)
            f = x < np.float32(1e-6)
            tl[k] = np.where(f, _interval(r[:, 1], lo, hi), x)
            fired[k] = f
        out.append((fired, tl.copy()))
    return out


def test_twin_equals_the_numpy_restatement():
    from oracle_lib import event_timers_init, event_timers_step
    seed, n, dt = 1234, 37, np.float32(0.1)
    ranges = [(0.5, 1.0), (0.0, 0.0), (0.1, 0.1), (0.02, 0.05), (2.0, 3.0), (0.3, 0.9), (0.0, 0.05), (1.0, 1.5)]
    rng = np.random.default_rng(0)
    dones = [(rng.random(n) < p).astype(np.uint8) for p in [0.0, 0.1, 1.0] + [0.05] * 37]
    for off in (0, 1000):
        for rr in (ranges[:1], ranges):
            want = _numpy_timers(seed, off, n, rr, dt, dones)
            tl = event_timers_init(seed, off, n, rr)
            fires = 0
            for t, done in enumerate(dones):
                fired = event_timers_step(seed, off, rr, dt, done, tl, t)
                assert np.array_equal(fired, want[t][0]), (off, t)
                assert np.array_equal(tl.view(np.uint32), want[t][1].view(np.uint32)), (off, t)
                fires += int(fired.sum())
            assert fires > 0
    # the semantics at the edges: lo == hi == 0 fires every step; a fresh timer of hi > step_dt never fires in its reset step
    tl = event_timers_init(seed, 0, n, [(0.0, 0.0), (0.5, 1.0)])
    fired = event_timers_step(seed, 0, [(0.0, 0.0), (0.5, 1.0)], dt, np.ones(n, np.uint8), tl, 5)
    assert fired[0].all() and not fired[1].any()


def test_twin_does_not_depend_on_sharding():
    from oracle_lib import event_timers_init, event_timers_step
    seed, n, dt, ranges = 7, 64, np.float32(0.1), [(0.1, 0.4), (0.0, 0.2)]
    rng = np.random.default_rng(1)
    whole = event_timers_init(seed, 0, n, ranges)
    halves = [event_timers_init(seed, 0, 32, ranges), event_timers_init(seed, 32, 32, ranges)]
    assert np.array_equal(whole, np.concatenate(halves, axis=1))
    for t in range(30):
        done = (rng.random(n) < 0.1).astype(np.uint8)
        f = event_timers_step(seed, 0, ranges, dt, done, whole, t)
        fh = [event_timers_step(seed, 32 * h, ranges, dt, done[32 * h:32 * h + 32], halves[h], t) for h in (0, 1)]
        assert np.array_equal(f, np.concatenate(fh, axis=1)) and np.array_equal(whole, np.concatenate(halves, axis=1))
