"""A modified policy observation group (DESIGN 6q) without a device: the CPU twin against a numpy restatement of IsaacLab's
ObservationManager.compute, the twin across shards, the cfg lowering and its refusals by term name, and the C-ABI's
argument checks."""
import ctypes as C
import sys
from pathlib import Path
from types import SimpleNamespace

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "tests"))

from oracle_lib import LIBRARY, policy_draw, policy_library, policy_observe  # noqa: E402

G = 16          # WL_NUM_GROUPS
SEED = 0x5EED1234ABCDEF


def _random_state(n, rng):
    st = rng.standard_normal((G, n, 4)).astype(np.float32)
    q = rng.standard_normal((n, 4))
    st[1] = (q / np.linalg.norm(q, axis=1, keepdims=True)).astype(np.float32)    # WL_G_QUAT: unit quaternions
    return st


def _restated(seed, env_id_offset, st, table, corrupt, t, call_idx):
    """ObservationManager.compute for one group, term by term: value, then noise (enable_corruption only), then clip, then
    scale, then the concatenation -- numpy fp32 arithmetic on the twin's library values and draws."""
    lib = policy_library(st)
    n = st.shape[1]
    blocks, j0 = [], 0
    for name, noise, clip, scale in table:
        first, width = LIBRARY[name]
        x = lib[:, first:first + width].copy()
        if corrupt and noise is not None:
            d = np.array([[policy_draw(seed, env_id_offset + i, t, call_idx, j0 + k, noise[0]) for k in range(width)] for i in range(n)],
                         dtype=np.float32)
            if noise[0] == "gaussian":                      # data + mean + std * randn_like(data)
                x = (x + np.float32(noise[1])) + np.float32(noise[2]) * d
            else:                                           # data + rand_like(data) * (n_max - n_min) + n_min
                x = (x + d * np.float32(noise[2] - noise[1])) + np.float32(noise[1])
        if clip is not None:
            x = np.minimum(np.maximum(x, np.float32(clip[0])), np.float32(clip[1]))
        if scale is not None:
            x = x * np.asarray(scale, dtype=np.float32)
        blocks.append(x.astype(np.float32))
        j0 += width
    return np.concatenate(blocks, axis=1)


TABLES = {
    "every_kind": [("root_pos_w", None, None, None), ("root_euler_xyz", None, None, None), ("base_lin_vel", None, None, None),
                   ("base_ang_vel", None, None, None), ("last_action", None, None, None), ("joint_vel", None, None, None),
                   ("joint_pos", None, None, None), ("wheel_friction", None, None, None), ("base_mass", None, None, None),
                   ("projected_gravity", None, None, None)],
    "noise_clip_scale": [("base_lin_vel", ("gaussian", 0.25, 0.5), (-0.7, 1.3), None),
                         ("projected_gravity", ("uniform", -0.05, 0.1), None, (1.0, -2.0, 0.5)),
                         ("root_euler_xyz", ("gaussian", -0.1, 0.2), None, 3.0),
                         ("joint_vel", ("uniform", -2.0, 1.0), (-1.5, 0.5), (0.5, 0.25, 2.0, 4.0)),
                         ("motor_damping", ("gaussian", 1.0, 0.3), (0.0, 2.0), 0.1)],
    "wide_32": [("projected_gravity", ("gaussian", 0.0, 0.05), None, None), ("base_ang_vel", ("gaussian", 0.0, 0.4), None, None),
                ("base_lin_vel", ("uniform", -0.5, 0.5), None, None), ("last_action", None, (-1.0, 1.0), None),
                ("joint_vel", ("gaussian", 0.1, 0.2), None, 0.01), ("joint_pos", ("uniform", 0.0, 0.1), (-0.3, 0.2), None),
                ("wheel_friction", ("gaussian", 0.0, 0.1), None, None), ("base_mass", ("uniform", -1.0, 1.0), None, 0.5),
                ("motor_damping", None, (-0.5, 0.5), (1.0, 2.0, 3.0, 4.0)), ("root_euler_xyz", ("gaussian", 0.0, 0.1), None, None),
                ("root_pos_w", None, None, None)],
}


def test_the_tables_cover_the_library():
    assert {t[0] for tb in TABLES.values() for t in tb} == set(LIBRARY)
    assert sum(LIBRARY[t[0]][1] for t in TABLES["wide_32"]) == 32


@pytest.mark.parametrize("table", sorted(TABLES))
@pytest.mark.parametrize("corrupt", [True, False])
@pytest.mark.parametrize("t,call_idx", [(0, -1), (12345, -1), (777, 0), (777, 5)])
def test_twin_equals_the_restated_observation_manager(table, corrupt, t, call_idx):
    rng = np.random.default_rng([sorted(TABLES).index(table), t, call_idx + 1])
    st = _random_state(37, rng)
    got = policy_observe(SEED, 5, st, TABLES[table], corrupt, t, call_idx)
    want = _restated(SEED, 5, st, TABLES[table], corrupt, t, call_idx)
    assert got.view(np.uint32).tolist() == want.view(np.uint32).tolist()


def test_the_draws_follow_the_documented_keys():
    """Gaussian columns below 12 share blind_obs's draws; the others differ across columns, steps and call indices."""
    g = lambda t, ci, j, k="gaussian": float(policy_draw(SEED, 3, t, ci, j, k))
    assert len({g(9, -1, 12), g(9, -1, 13), g(9, -1, 16), g(10, -1, 12), g(9, 0, 12), g(9, 1, 12)}) == 6
    assert len({g(9, -1, j, "uniform") for j in range(32)} | {g(9, 0, 0, "uniform"), g(10, -1, 0, "uniform")}) == 34
    assert g(9, -1, 0) != g(9, 0, 0) != g(9, 1, 0)


def test_twin_does_not_depend_on_sharding():
    rng = np.random.default_rng(3)
    st = _random_state(64, rng)
    table = TABLES["wide_32"]
    whole = policy_observe(SEED, 0, st, table, True, 41, -1)
    halves = np.concatenate([policy_observe(SEED, 0, st[:, :32], table, True, 41, -1), policy_observe(SEED, 32, st[:, 32:], table, True, 41, -1)])
    assert whole.view(np.uint32).tolist() == halves.view(np.uint32).tolist()


# ---- the cfg lowering ------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def ref_registry():
    if str(ROOT / "shims") not in sys.path:
        sys.path.insert(0, str(ROOT / "shims"))
    import recorded_cfgs
    return recorded_cfgs.load()


def _named(name):
    f = lambda env, **kw: None
    f.__name__ = name
    return f


def _drift_cfg(reg, gid="Isaac-MushrDriftRL-v0", **terms):
    cfg = reg[gid]["cfgs"]["env_cfg_entry_point"]()
    cfg.scene.num_envs = 16
    if terms:
        from isaaclab.managers import ObservationTermCfg
        old = cfg.observations.policy
        g = SimpleNamespace(concatenate_terms=True, enable_corruption=getattr(old, "enable_corruption", False))
        for k, v in terms.items():
            setattr(g, k, v if hasattr(v, "func") else ObservationTermCfg(func=v))
        cfg.observations.policy = g
    return cfg


def test_drift_without_root_pos_w_lowers_to_an_11_float_table_with_the_flag_only(ref_registry):
    from wheeledlab_b200 import policy_obs
    from wheeledlab_b200.compat import spec_from_reference_cfg
    for gid in ("Isaac-MushrDriftRL-v0", "Isaac-F1TenthDriftRL-v0"):
        cfg = _drift_cfg(ref_registry, gid)
        pol = cfg.observations.policy
        want = [(n, getattr(pol, n)) for n in ("root_euler_xyz_term", "base_lin_vel_term", "base_ang_vel_term", "last_action_term")]
        pol.root_pos_w_term = None
        with pytest.raises(NotImplementedError, match="differ"):
            spec_from_reference_cfg(cfg)
        spec = spec_from_reference_cfg(cfg, device_terms=True)
        plain = spec_from_reference_cfg(_drift_cfg(ref_registry, gid))
        assert policy_obs.row_width([t[1:] for t in spec.policy_terms]) == 11 and spec.obs_dim == 14
        assert [t[0] for t in spec.policy_terms] == [n for n, _ in want]
        assert [t[1] for t in spec.policy_terms] == ["root_euler_xyz", "base_lin_vel", "base_ang_vel", "last_action"]
        for (_, term), (_, _, noise, clip, scale) in zip(want, spec.policy_terms):
            n = getattr(term, "noise", None)
            assert noise == (None if n is None else ("gaussian", float(n.mean), float(n.std)))
            assert clip == (None if term.clip is None else tuple(float(x) for x in term.clip)) and scale is None
        assert bytes(spec.cfg) == bytes(plain.cfg), "the built-in row's config is left as the task's"


def test_unmodified_cfgs_lower_to_the_committed_blobs_with_no_table(ref_registry):
    from wheeledlab_b200.compat import spec_from_reference_cfg
    blobs = ROOT / "tests" / "golden" / "cfg_blobs"
    for gid in ("Isaac-MushrDriftRL-v0", "Isaac-F1TenthDriftRL-v0"):
        for key, suffix in (("env_cfg_entry_point", "ref"), ("play_env_cfg_entry_point", "play.ref")):
            make_cfg = ref_registry[gid]["cfgs"].get(key)
            if make_cfg is None:
                continue
            for flag in (False, True):
                cfg = make_cfg(); cfg.scene.num_envs = 4096
                got = spec_from_reference_cfg(cfg, device_terms=flag)
                assert got.policy_terms == []
                assert C.string_at(C.addressof(got.cfg), C.sizeof(got.cfg)) == (blobs / f"{gid}.{suffix}.bin").read_bytes(), (gid, key, flag)


def test_compat_refuses_what_the_policy_kernel_does_not_do_by_term_name(ref_registry):
    from isaaclab.managers import ObservationTermCfg, SceneEntityCfg
    from isaaclab.utils.noise import AdditiveGaussianNoiseCfg
    from wheeledlab_b200.compat import spec_from_reference_cfg
    keep = {"yaw": _named("root_euler_xyz")}
    bad = {
        "lidar": (ObservationTermCfg(func=_named("lidar_ranges")), NotImplementedError, "not in the policy observation library"),
        "laplace_vel": (ObservationTermCfg(func=_named("base_lin_vel"), noise=SimpleNamespace(b=0.1)), NotImplementedError, "noise model"),
        "scaled_noise": (ObservationTermCfg(func=_named("base_lin_vel"), noise=AdditiveGaussianNoiseCfg(std=0.1, operation="scale")),
                         NotImplementedError, "operation"),
        "filtered": (ObservationTermCfg(func=_named("base_ang_vel"), modifiers=[object()]), NotImplementedError, "modifiers"),
        "steer_rate": (ObservationTermCfg(func=_named("joint_vel"), params={"asset_cfg": SceneEntityCfg("robot", joint_names=[".*_steer"])}),
                       NotImplementedError, "throttle joints only"),
        "wheel_angle": (ObservationTermCfg(func=_named("joint_pos"), params={"asset_cfg": SceneEntityCfg("robot", joint_names=[".*_throttle"])}),
                        NotImplementedError, "steer joints only"),
        "inf_clip": (ObservationTermCfg(func=_named("last_action"), clip=(-float("inf"), 1.0)), ValueError, "not finite"),
    }
    for name, (term, exc, msg) in bad.items():
        with pytest.raises(exc, match=msg) as e:
            spec_from_reference_cfg(_drift_cfg(ref_registry, **keep, **{name: term}), device_terms=True)
        assert name in str(e.value)
    cfg = _drift_cfg(ref_registry, **keep)
    cfg.observations.policy.concatenate_terms = False
    with pytest.raises(NotImplementedError, match="concatenate_terms"):
        spec_from_reference_cfg(cfg, device_terms=True)
    wide = {f"spin{k}": _named("joint_vel") for k in range(9)}             # 36 floats
    with pytest.raises(NotImplementedError, match="36 floats") as e:
        spec_from_reference_cfg(_drift_cfg(ref_registry, **wide), device_terms=True)
    assert "spin8" in str(e.value)
    for gid, task in (("Isaac-MushrElevationRL-v0", "Elevation"), ("Isaac-MushrVisualRL-v0", "Visual")):
        cfg = ref_registry[gid]["cfgs"]["env_cfg_entry_point"]()
        cfg.scene.num_envs = 16
        cfg.observations.policy.base_lin_vel = None
        with pytest.raises(NotImplementedError, match=task):
            spec_from_reference_cfg(cfg, device_terms=True)


def test_c_abi_argument_checks_need_no_device():
    import wheeledlab_b200 as wl
    from wheeledlab_b200._lib import WlPolicyTerm
    lib = wl.lib
    assert lib.wl_set_policy_terms(None, None, 0) < 0 and b"null handle" in lib.wl_last_error()
    assert lib.wl_policy_obs_dim(None) == 0
    assert lib.wl_policy_observe(None, 0, -1, None, None) < 0 and b"null argument" in lib.wl_last_error()
    assert C.sizeof(WlPolicyTerm) == 80 and WlPolicyTerm.scale.offset == 48
