"""Noise, clip and scale on the Elevation and Visual rows (DESIGN 6r) without a device: the oracle twin against the built-in
rows and against a numpy restatement of IsaacLab's ObservationManager.compute, the twin across shards, the cfg lowering
and its refusals by term name, and the C-ABI's argument checks."""
import ctypes as C
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "tests"))

import oracle_lib as O  # noqa: E402
import row_terms_oracle as R  # noqa: E402

SEED = 0x5EED1234ABCDEF
ELEV = ("goal_relative_xyz", "root_euler_xyz", "base_lin_vel", "base_ang_vel", "last_action", "world_height_map")
VIS = ("base_lin_vel", "base_ang_vel", "last_action")


def _spec(task, n, corrupt=0, env_id_offset=0):
    import wheeledlab_b200 as wl
    spec = wl.elevation_task(num_envs=n, seed=11, env_id_offset=env_id_offset) if task == "elevation" else \
        wl.visual_task(num_envs=n, seed=11, env_id_offset=env_id_offset)
    spec.cfg.enable_corruption = corrupt
    return spec


def _randomise(o, spec, rng):
    """Random states: positions over the raster and beyond it (ray misses), unit quaternions, velocities past the clips,
    actions past +-1, goals anywhere."""
    st = o.export_state()
    n, c = st.shape[1], spec.cfg
    if int(c.task) == 1:
        x1, y1 = c.hf_x0 + c.hf_nx * c.hf_cell, c.hf_y0 + c.hf_ny * c.hf_cell
        st[0, :, 0] = rng.uniform(c.hf_x0 - 3.0, x1 + 3.0, n)
        st[0, :, 1] = rng.uniform(c.hf_y0 - 3.0, y1 + 3.0, n)
        st[0, :, 2] = rng.uniform(-0.5, 1.5, n)
        st[14, :, :2] = rng.uniform(-30.0, 30.0, (n, 2))                       # WL_G_CMDB
    q = rng.standard_normal((n, 4))
    st[1] = (q / np.linalg.norm(q, axis=1, keepdims=True)).astype(np.float32)
    st[2, :, :3] = rng.uniform(-25.0, 25.0, (n, 3))
    st[3, :, :3] = rng.uniform(-25.0, 25.0, (n, 3))
    st[6, :, :2] = rng.uniform(-2.0, 2.0, (n, 2))
    o.import_state(st)


def _oracle(task, n, corrupt=0, env_id_offset=0, seed=0):
    spec = _spec(task, n, corrupt, env_id_offset)
    o = R.RowOracle(spec.cfg, heightfield=spec.heightfield)
    o.startup(); o.reset(None, 0)
    _randomise(o, spec, np.random.default_rng(seed))
    return spec, o


def _registered(task, clip=10.0):
    from wheeledlab_b200 import row_terms
    return row_terms.registered(task, clip)


def test_registered_row_terms_are_the_built_in_rows():
    for task in ("elevation", "visual"):
        spec, o = _oracle(task, 64, seed=1)
        builtin = o.observe(17, 2)
        twin = o.row_observe(_registered(task, spec.cfg.obs_clip), 17, 2, obs=builtin.copy())
        assert twin.view(np.uint32).tolist() == builtin.view(np.uint32).tolist(), task
        if task == "elevation":
            raw = o.row_raw()
            assert np.isinf(raw[:, 13:]).any() and np.isfinite(raw[:, 13:]).any(), "the states include ray misses and hits"


def _clamp(x, lo, hi):
    v = np.where(x > np.float32(lo), x, np.float32(lo))
    return np.where(v < np.float32(hi), v, np.float32(hi)).astype(np.float32)


def _restated(o, terms, t, call_idx, corrupt):
    """ObservationManager.compute term by term on the twin's raw values and draws: value, noise (enable_corruption only),
    clip, scale -- numpy fp32 arithmetic, the parameters rounded to fp32 (a uniform span formed in double)."""
    raw = o.row_raw()
    n, out, j0 = raw.shape[0], [], 0
    gid0 = int(o.cfg.env_id_offset)
    for name, noise, clip, scale in terms:
        w = R.ROW_KINDS[name][1]
        x = raw[:, j0:j0 + w].copy()
        if corrupt and noise is not None:
            d = np.array([[R.row_draw(int(o.cfg.seed), gid0 + i, t, call_idx, j0 + k, noise[0]) for k in range(w)]
                          for i in range(n)], dtype=np.float32)
            if noise[0] == "gaussian":                          # data + mean + std * randn_like(data)
                x = (x + np.float32(noise[1])) + np.float32(noise[2]) * d
            else:                                               # data + rand_like(data) * (n_max - n_min) + n_min
                x = (x + d * np.float32(float(noise[2]) - float(noise[1]))) + np.float32(noise[1])
        if clip is not None:
            x = _clamp(x, clip[0], clip[1])
        if scale is not None:
            x = x * np.asarray(scale if isinstance(scale, tuple) else (scale,), dtype=np.float32)
        out.append(x.astype(np.float32))
        j0 += w
    return np.concatenate(out, axis=1)


ELEV_TERMS = [
    ("goal_relative_xyz", ("gaussian", 0.25, 0.5), (-3.0, 7.0), (2.0, -0.5)),
    ("root_euler_xyz", ("uniform", -0.2, 0.6), None, 1.5),
    ("base_lin_vel", ("gaussian", -0.1, 0.3), (-4.0, 2.5), None),
    ("base_ang_vel", None, (-10.0, 10.0), (0.5, 1.0, -2.0)),
    ("last_action", ("uniform", 0.05, 0.15), (-1.0, 1.0), None),
    ("world_height_map", ("uniform", -0.1, 0.3), None, 0.7),
]
ELEV_TERMS_G = ELEV_TERMS[:5] + [("world_height_map", ("gaussian", 0.02, 0.05), (-0.3, 0.9), 2.0)]
VIS_TERMS = [("base_lin_vel", ("uniform", -0.1, 0.1), None, (1.0, 2.0, 3.0)),
             ("base_ang_vel", ("gaussian", 0.3, 0.2), (-2.0, 5.0), None),
             ("last_action", ("uniform", -0.1, 0.1), (-1.0, 1.0), 0.5)]


@pytest.mark.parametrize("task,terms", [("elevation", ELEV_TERMS), ("elevation", ELEV_TERMS_G), ("visual", VIS_TERMS)])
@pytest.mark.parametrize("corrupt,t,call_idx", [(1, 41, -1), (1, 7, 3), (0, 41, -1)])
def test_twin_equals_the_restated_observation_manager(task, terms, corrupt, t, call_idx):
    spec, o = _oracle(task, 6, corrupt=corrupt, seed=2)
    twin = o.row_observe(terms, t, call_idx)
    tail = twin[:, -8:] if task == "visual" else twin
    want = _restated(o, terms, t, call_idx, corrupt)
    assert tail.view(np.uint32).tolist() == want.view(np.uint32).tolist()
    if task == "elevation" and terms is ELEV_TERMS:
        assert np.isposinf(twin[:, 13:]).any(), "a miss without a clip stays +inf"
    if task == "elevation" and terms is ELEV_TERMS_G:
        assert np.isfinite(twin[:, 13:]).all() and (twin[:, 13:] == np.float32(0.9 * 2.0)).any(), "a clipped miss is the clip"


def test_the_draws_follow_the_documented_keys():
    for kind, off in (("gaussian", 0), ("uniform", 256)):
        for j, call in ((0, -1), (13, -1), (688, 4), (5, 0)):
            w = O.philox(SEED, 9, 123, 17, 512 * (call + 1) + off + j // 4, 1).reshape(4)
            d = R.row_draw(SEED, 9, 123, call, j, kind)
            if kind == "uniform":
                assert d == np.float32((int(w[j % 4]) >> 8) * 5.9604644775390625e-08)
            else:
                assert np.isfinite(d)
    # a Gaussian and a uniform column of the same block take different words
    assert R.row_draw(SEED, 1, 2, -1, 12, "uniform") != R.row_draw(SEED, 1, 2, -1, 12, "gaussian")


def test_twin_does_not_depend_on_sharding():
    import wheeledlab_b200 as wl  # noqa: F401
    for task, terms in (("elevation", ELEV_TERMS), ("visual", VIS_TERMS)):
        spec, whole = _oracle(task, 16, corrupt=1, seed=3)
        st = whole.export_state()
        rows = whole.row_observe(terms, 29, -1)
        parts = []
        for off in (0, 8):
            sp = _spec(task, 8, 1, env_id_offset=off)
            o = R.RowOracle(sp.cfg, heightfield=sp.heightfield)
            o.startup()
            o.import_state(np.ascontiguousarray(st[:, off:off + 8]))
            parts.append(o.row_observe(terms, 29, -1))
        assert rows.view(np.uint32).tolist() == np.concatenate(parts).view(np.uint32).tolist(), task


# ---- the cfg lowering ------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def ref_registry():
    if str(ROOT / "shims") not in sys.path:
        sys.path.insert(0, str(ROOT / "shims"))
    import recorded_cfgs
    return recorded_cfgs.load()


def _cfg(reg, gid, key="env_cfg_entry_point", n=16):
    cfg = reg[gid]["cfgs"][key]()
    cfg.scene.num_envs = n
    return cfg


def test_corrupted_visual_cfg_lowers_to_three_uniform_row_terms_with_the_flag_only(ref_registry):
    from wheeledlab_b200.compat import spec_from_reference_cfg
    from isaaclab.utils.noise import AdditiveUniformNoiseCfg
    gid = "Isaac-MushrVisualRL-v0"
    cfg = _cfg(ref_registry, gid)
    cfg.observations.policy.enable_corruption = True
    # the cfg writes last_action's noise as Unoise(-.1, .1): positional, so the two numbers are not n_min / n_max
    with pytest.raises(NotImplementedError, match="operation") as e:
        spec_from_reference_cfg(cfg, device_terms=True)
    assert "last_action" in str(e.value)
    cfg.observations.policy.last_action.noise = AdditiveUniformNoiseCfg(n_min=-0.1, n_max=0.1)
    spec = spec_from_reference_cfg(cfg, device_terms=True)
    assert [t[:2] for t in spec.row_terms] == [("base_lin_vel", "base_lin_vel"), ("base_ang_vel", "base_ang_vel"), ("last_action", "last_action")]
    assert [t[2] for t in spec.row_terms] == [("uniform", -0.1, 0.1)] * 3
    assert [t[3] for t in spec.row_terms] == [None, None, (-1.0, 1.0)] and all(t[4] is None for t in spec.row_terms)
    plain = spec_from_reference_cfg(cfg)
    assert plain.row_terms == []
    ref = spec_from_reference_cfg(_cfg(ref_registry, gid))
    ref.cfg.enable_corruption = 1
    assert bytes(plain.cfg) == bytes(ref.cfg), "without the flag the spec is what it was"


def test_elevation_map_noise_lowers_to_row_terms(ref_registry):
    from isaaclab.utils.noise import AdditiveUniformNoiseCfg
    from wheeledlab_b200.compat import spec_from_reference_cfg
    cfg = _cfg(ref_registry, "Isaac-MushrElevationRL-v0")
    cfg.observations.policy.enable_corruption = True
    cfg.observations.policy.elevation_map.noise = AdditiveUniformNoiseCfg(n_min=-0.05, n_max=0.05)
    spec = spec_from_reference_cfg(cfg, device_terms=True)
    assert [t[1] for t in spec.row_terms] == list(ELEV)
    assert spec.row_terms[5][2:] == (("uniform", -0.05, 0.05), (-10.0, 10.0), None)
    assert [t[3] for t in spec.row_terms[:5]] == [None, None, (-10.0, 10.0), (-10.0, 10.0), (-1.0, 1.0)]
    assert spec_from_reference_cfg(cfg).row_terms == []
    cfg.observations.policy.enable_corruption = False                   # noise without corruption: the built-in row
    assert spec_from_reference_cfg(cfg, device_terms=True).row_terms == []
    cfg.observations.policy.base_ang_vel.clip = (-5.0, 5.0)             # per-term clips: no longer one shared clip
    spec = spec_from_reference_cfg(cfg, device_terms=True)
    assert [t[3] for t in spec.row_terms] == [None, None, (-10.0, 10.0), (-5.0, 5.0), (-1.0, 1.0), (-10.0, 10.0)]


def test_registered_cfgs_lower_to_the_committed_blobs_with_no_row_terms(ref_registry):
    from wheeledlab_b200.compat import spec_from_reference_cfg
    blobs = ROOT / "tests" / "golden" / "cfg_blobs"
    for gid in ("Isaac-MushrElevationRL-v0", "Isaac-MushrVisualRL-v0"):
        for key, suffix in (("env_cfg_entry_point", "ref"), ("play_env_cfg_entry_point", "play.ref")):
            if ref_registry[gid]["cfgs"].get(key) is None:
                continue
            for flag in (False, True):
                cfg = _cfg(ref_registry, gid, key, n=4096)
                got = spec_from_reference_cfg(cfg, device_terms=flag)
                assert got.row_terms == []
                if "Visual" in gid:              # the reference draws a new random traversability map at every import
                    got.cfg.vis_n_trav = int(np.load(blobs / "visual_ref_map.npz")["map"].sum())
                assert C.string_at(C.addressof(got.cfg), C.sizeof(got.cfg)) == (blobs / f"{gid}.{suffix}.bin").read_bytes(), (gid, key, flag)


def test_compat_refuses_what_the_row_kernels_do_not_do_by_term_name(ref_registry):
    from types import SimpleNamespace
    from isaaclab.utils.noise import AdditiveGaussianNoiseCfg, AdditiveUniformNoiseCfg
    from wheeledlab_b200.compat import spec_from_reference_cfg
    bad = {
        "base_lin_vel": ("noise", SimpleNamespace(b=0.1), NotImplementedError, "noise model"),
        "base_ang_vel": ("noise", AdditiveGaussianNoiseCfg(std=0.1, operation="scale"), NotImplementedError, "operation"),
        "last_action": ("modifiers", [object()], NotImplementedError, "modifiers"),
        "world_euler_xyz": ("history_length", 3, NotImplementedError, "history_length"),
        "elevation_map": ("scale", tuple([1.0] * 676), NotImplementedError, "per-element scale"),
        "goal_relative_xyz": ("clip", (-float("inf"), 1.0), ValueError, "not finite"),
    }
    for name, (attr, value, exc, msg) in bad.items():
        cfg = _cfg(ref_registry, "Isaac-MushrElevationRL-v0")
        cfg.observations.policy.enable_corruption = True
        cfg.observations.policy.elevation_map.noise = AdditiveUniformNoiseCfg(n_min=-0.05, n_max=0.05)
        setattr(getattr(cfg.observations.policy, name), attr, value)
        with pytest.raises(exc, match=msg) as e:
            spec_from_reference_cfg(cfg, device_terms=True)
        assert name in str(e.value)
    cfg = _cfg(ref_registry, "Isaac-MushrVisualRL-v0")
    cfg.observations.policy.enable_corruption = True
    cfg.observations.policy.camera.scale = 2.0
    with pytest.raises(NotImplementedError, match="camera"):
        spec_from_reference_cfg(cfg, device_terms=True)


def test_env_refuses_a_term_list_other_than_the_rows_own():
    from wheeledlab_b200 import row_terms
    row_terms.check_order("elevation", ELEV)
    row_terms.check_order("visual", VIS)
    for task, fns in (("elevation", ELEV[:5]), ("elevation", ELEV[1:] + ELEV[:1]), ("visual", ("base_ang_vel", "base_lin_vel", "last_action"))):
        with pytest.raises(NotImplementedError, match="modified term list"):
            row_terms.check_order(task, fns)
    with pytest.raises(NotImplementedError, match="Drift"):
        row_terms.task_terms("drift")
    assert row_terms.is_builtin("elevation", row_terms.registered("elevation", 4.0))
    assert row_terms.is_builtin("visual", row_terms.registered("visual"))


def test_c_abi_argument_checks_need_no_device():
    import wheeledlab_b200 as wl
    from wheeledlab_b200._lib import WL_ROW_TERMS, WlPolicyTerm
    lib = wl.lib
    assert lib.wl_set_row_terms(None, None, 0) < 0 and b"null handle" in lib.wl_last_error()
    assert lib.wl_row_terms(None) == 0
    assert C.sizeof(WlPolicyTerm) == C.sizeof(R.PolicyTerm) == 80
    assert {k: v[0] for k, v in WL_ROW_TERMS.items()} == {k: v[0] for k, v in R.ROW_KINDS.items()}
