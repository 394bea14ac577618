"""Device terms without a device: the registry (module AND name identify a reference function), the parameters it
folds, the argument refusals of the C entries on a null handle, and compat's lowering with device_terms=False / True."""
import ctypes as C
import types

import pytest


def _fake(module, name):
    def f(env, **kw):
        return None
    f.__module__, f.__name__ = module, name
    return f


def test_same_name_in_elevation_and_visual_maps_to_different_kinds():
    from wheeledlab_b200 import device_terms as dtm
    e = dtm.lookup(_fake("wheeledlab_tasks.elevation.mushr_elevation_env_cfg", "forward_vel"))
    assert e is not None and e.kind == 1
    assert dtm.lookup(_fake("wheeledlab_tasks.visual.mushr_visual_env_cfg", "forward_vel")) is None   # built in, not a device term
    assert dtm.lookup(_fake("wheeledlab_tasks.visual.mushr_visual_env_cfg", "off_track")).kind == 15
    assert dtm.lookup(_fake("wheeledlab_tasks.drifting.mushr_drift_env_cfg", "off_track")) is None
    assert dtm.lookup(_fake("wheeledlab_tasks.elevation.mushr_elevation_env_cfg", "upright_bool")) is None
    assert dtm.lookup(lambda env: None) is None
    assert dtm.lookup(_fake("somewhere.else", "ascending")) is None
    kinds = [k.kind for k in dtm.REGISTRY.values()]
    assert sorted(kinds) == list(range(1, 18)) and len(set(dtm.REGISTRY)) == 17


def test_parameters_follow_the_reference_defaults_and_refuse_what_it_would():
    from wheeledlab_b200 import device_terms as dtm
    vr = dtm.resolve("vel_rew_trav", dtm.VISUAL)
    assert dtm.param_values(vr, {}) == [1.0, 2.0, 0.0, 0.0]
    assert dtm.param_values(vr, {"speed_target_on_non_trav": 3}) == [1.0, 3.0, 0.0, 0.0]
    with pytest.raises(TypeError, match="missing"):
        dtm.param_values(dtm.resolve("steep_penalty", dtm.ELEVATION), {})
    with pytest.raises(TypeError, match="unexpected"):
        dtm.param_values(dtm.resolve("ascending", dtm.ELEVATION), {"x": 1})
    with pytest.raises(ValueError):
        dtm.param_values(dtm.resolve("low_vel_penalty", dtm.ELEVATION), {"min_vel": float("inf")})
    assert [k.name for k in dtm.REGISTRY.values() if k.map_term] == ["is_traversable", "is_traversable_speed_scaled", "vel_rew_trav",
                                                                      "bool_is_not_traversable"]


def test_device_term_entries_refuse_a_null_handle_without_a_device():
    import wheeledlab_b200 as wl
    from wheeledlab_b200._lib import WlTermDesc
    d = (WlTermDesc * 1)(WlTermDesc(1, 0, 1.0, (C.c_double * 4)()))
    assert wl.lib.wl_set_device_terms(None, d, 1) == -1
    p = C.c_void_p(1 << 20)
    assert wl.lib.wl_step_terms(None, p, p, p, p, p, None, None, 0, None) == -1
    assert wl.lib.wl_device_term_masks(None) is None
    assert C.sizeof(WlTermDesc) == 48


def test_step_host_and_mixing_are_refused_by_the_env_before_any_device_work():
    from wheeledlab_b200.env import ManagerBasedRLEnv
    env = types.SimpleNamespace(_py_rewards=[types.SimpleNamespace(name="py")], _py_terms=[], _dev_terms=[])
    with pytest.raises(NotImplementedError, match="not both"):
        ManagerBasedRLEnv._refuse_mixing(env, device=True)
    env = types.SimpleNamespace(_py_rewards=[], _py_terms=[], _dev_terms=[types.SimpleNamespace(name="d")])
    with pytest.raises(NotImplementedError, match="not both"):
        ManagerBasedRLEnv._refuse_mixing(env)
    with pytest.raises(NotImplementedError, match="step_host"):
        ManagerBasedRLEnv.step_host(env, None)


def test_compat_device_terms_lowering():
    """device_terms=False: today's spec and blob exactly; True: the cfg's library terms become device terms in cfg order,
    with its weights and params, and the config blob is the same; a function outside the library still raises or
    becomes a Python term."""
    import sys
    from pathlib import Path
    root = Path(__file__).resolve().parent.parent
    if str(root / "shims") not in sys.path:
        sys.path.insert(0, str(root / "shims"))
    import recorded_cfgs
    from isaaclab.managers import RewardTermCfg, TerminationTermCfg
    from wheeledlab_b200.compat import spec_from_reference_cfg
    E = recorded_cfgs.load()["Isaac-MushrElevationRL-v0"]["cfgs"]["env_cfg_entry_point"]
    blob = lambda c: C.string_at(C.addressof(c), C.sizeof(c))
    mod = "wheeledlab_tasks.elevation.mushr_elevation_env_cfg"
    steep, up, asc = _fake(mod, "steep_penalty"), _fake(mod, "upright_penalty"), _fake(mod, "ascending")
    base = E(); base.scene.num_envs = 8
    plain = spec_from_reference_cfg(base)
    assert blob(spec_from_reference_cfg(base, device_terms=False).cfg) == blob(plain.cfg)
    cfg = E(); cfg.scene.num_envs = 8
    cfg.rewards.steep = RewardTermCfg(func=steep, weight=-2.0, params={"thresh_pitch": 0.4})
    cfg.rewards.asc = RewardTermCfg(func=asc, weight=3.0)
    cfg.terminations.tilt = TerminationTermCfg(func=up, params={"thresh_deg": 50.0}, time_out=True)
    for group, names in ((cfg.rewards, ["steep", "asc"]), (cfg.terminations, ["tilt"])):
        if hasattr(group, "_cfg_fields"):
            group._cfg_fields = list(group._cfg_fields) + names
    with pytest.raises(NotImplementedError):
        spec_from_reference_cfg(cfg)
    with pytest.raises(NotImplementedError):
        spec_from_reference_cfg(cfg, device_terms=False)
    s = spec_from_reference_cfg(cfg, device_terms=True)
    assert s.device_terms == [("steep", steep, "reward", -2.0, {"thresh_pitch": 0.4}), ("asc", asc, "reward", 3.0, {}),
                              ("tilt", up, "time_out", 0.0, {"thresh_deg": 50.0})]
    assert s.python_reward_terms == [] and s.python_termination_terms == []
    assert blob(s.cfg) == blob(plain.cfg) and s.reward_names == plain.reward_names
    cfg.rewards.other = RewardTermCfg(func=lambda env: 0, weight=1.0)
    if hasattr(cfg.rewards, "_cfg_fields"):
        cfg.rewards._cfg_fields = list(cfg.rewards._cfg_fields) + ["other"]
    with pytest.raises(NotImplementedError, match="allow_python_terms"):
        spec_from_reference_cfg(cfg, device_terms=True)
    s = spec_from_reference_cfg(cfg, device_terms=True, allow_python_terms=True)
    assert [t[0] for t in s.python_reward_terms] == ["other"] and len(s.device_terms) == 3


def test_compat_routes_a_library_function_before_the_built_in_slot_of_the_same_name():
    """The Elevation forward_vel (clamped at 1.2) on the Visual cfg is a device term, not the Visual built-in forward_vel
    (unclamped): the built-in slot keeps the cfg's own vel_rew weight."""
    import sys
    from pathlib import Path
    root = Path(__file__).resolve().parent.parent
    if str(root / "shims") not in sys.path:
        sys.path.insert(0, str(root / "shims"))
    import recorded_cfgs
    from isaaclab.managers import RewardTermCfg
    from wheeledlab_b200.compat import spec_from_reference_cfg
    Vc = recorded_cfgs.load()["Isaac-MushrVisualRL-v0"]["cfgs"]["env_cfg_entry_point"]
    blob = lambda c: C.string_at(C.addressof(c), C.sizeof(c))
    plain_cfg = Vc(); plain_cfg.scene.num_envs = 8
    plain = spec_from_reference_cfg(plain_cfg)
    fv = _fake("wheeledlab_tasks.elevation.mushr_elevation_env_cfg", "forward_vel")
    cfg = Vc(); cfg.scene.num_envs = 8
    cfg.rewards.fv_elev = RewardTermCfg(func=fv, weight=4.0)
    if hasattr(cfg.rewards, "_cfg_fields"):
        cfg.rewards._cfg_fields = list(cfg.rewards._cfg_fields) + ["fv_elev"]
    s = spec_from_reference_cfg(cfg, device_terms=True)
    assert s.device_terms == [("fv_elev", fv, "reward", 4.0, {})]
    assert list(s.cfg.rew_weight)[1] == list(plain.cfg.rew_weight)[1] == 7.0
    assert blob(s.cfg) == blob(plain.cfg) and s.reward_names == plain.reward_names
