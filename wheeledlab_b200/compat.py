"""Lowering of the REFERENCE's own env-cfg objects onto the fused kernels' POD config.

``gym.make("Isaac-MushrDriftRL-v0", cfg=env_cfg)`` hands the unmodified ``MushrDriftRLEnvCfg`` /
``MushrElevationRLEnvCfg`` / ``F1TenthDriftRLEnvCfg`` instance (built against IsaacLab, or against the stand-in in
``shims/isaaclab``) to the entry point.  This module reads that object -- terms are recognised by the NAME of the
function they reference, values are taken from the cfg (weights, params, dt, decimation, scales, noise, DR ranges) --
and fills a ``TaskSpec``.  A term the kernels do not implement raises ``NotImplementedError`` (no silent fallback); the
observation group is validated term by term (function, order, clip; BlindObs noise stds are read from the cfg).  A ``critic``
group next to ``policy`` (Drift family) is lowered to the term table of the critic observation kernel (privileged.py).

Reference files: wheeledlab_tasks/drifting/mushr_drift_env_cfg.py, f1tenth_drift_env_cfg.py,
elevation/mushr_elevation_env_cfg.py, common/{actions,observations}.py.
"""
from __future__ import annotations

import math

from . import tasks as T

_DRIFT_REWARDS = {"side_slip": 0, "vel_dist": 1, "track_progress_rate": 2, "turn_left_go_right": 3, "energy_through_turn": 4,
                  "cross_track_dist": 5, "is_terminated_term": 6}
_ALIASES = {"turn_left_go_right_f1": "turn_left_go_right"}    # f1tenth_drift_env_cfg.py:90-104: same math, other joint names
_ELEV_REWARDS = {"goal_progress_rate": 0, "higher_elevation": 1, "is_falling_penalty": 2, "is_terminated_term": 3}
_VIS_REWARDS = {"traversable_reward": 0, "forward_vel": 1}
_ACTION_KINDS = {"RCCarRWDAction": T.ACT_RWD, "RCCar4WDAction": T.ACT_4WD, "AckermannAction": T.ACT_ACKERMANN}
# observation groups the kernels implement: term functions in order (common/observations.py:19-56,
# elevation/mushr_elevation_env_cfg.py:57-88, visual/mushr_visual_env_cfg.py:37-57)
_OBS_BLIND = ["root_pos_w", "root_euler_xyz", "base_lin_vel", "base_ang_vel", "last_action"]
_OBS_ELEV = ["goal_relative_xyz", "root_euler_xyz", "base_lin_vel", "base_ang_vel", "last_action", "world_height_map"]
_OBS_VIS_TAIL = ["base_lin_vel", "base_ang_vel", "last_action"]
_CAMERA_FUNCS = {"camera_data_rgb_flattened_aug": "aug", "camera_data_rgb_flattened": "raw"}
_BOUND = {None: T.BOUND_NONE, "clip": T.BOUND_CLIP, "tanh": T.BOUND_TANH}
_RESET_EVENTS = ("material", "actuator_gains", "base_mass", "wheel_mass")     # the WL_RESET_EV_* bits, in bit order


def _fields(obj):
    if obj is None:
        return []
    names = getattr(obj, "_cfg_fields", None) or [k for k in vars(obj) if not k.startswith("_")]
    return [(k, getattr(obj, k)) for k in names if getattr(obj, k) is not None]


def _fname(term):
    f = term.func
    return getattr(f, "__name__", type(f).__name__)


def _obs_funcs(cfg):
    return [_fname(t) for _, t in _fields(cfg.observations.policy) if hasattr(t, "func")]


def _task_kind(cfg) -> str:
    """Which kernel family a reference env cfg maps to, decided by its observation group (present in train AND play cfgs)."""
    funcs = _obs_funcs(cfg)
    if "world_height_map" in funcs:
        return "elevation"
    if any(f in _CAMERA_FUNCS for f in funcs):
        return "visual"
    if "root_pos_w" in funcs:
        return "drift"
    from ._lib import WL_POLICY_TERMS
    if any(f in WL_POLICY_TERMS for f in funcs):           # a modified Drift group (lowered with device_terms only)
        return "drift"
    raise NotImplementedError(f"observation group {funcs} is not one the fused step implements")


def _validate_obs(cfg, expected, c, blind=False, task=None):
    """The observation group must be exactly what the kernel assembles: same term functions in the same order; noise stds
    (BlindObs) and clips are read from the cfg."""
    terms = [(k, t) for k, t in _fields(cfg.observations.policy) if hasattr(t, "func")]
    funcs = [_fname(t) for _, t in terms]
    if funcs != expected:
        raise NotImplementedError(f"observation terms {funcs} differ from the kernel's {expected} (order matters)"
                                  + (f"; a modified {task} policy group is not implemented (the policy observation table covers "
                                     "the Drift family)" if task else ""))
    if getattr(cfg.observations.policy, "concatenate_terms", True) is not True:
        raise NotImplementedError("observation group must concatenate its terms")
    for k, (name, t) in enumerate(terms):
        fn = funcs[k]
        clip = getattr(t, "clip", None)
        if fn == "last_action":
            if clip is not None and tuple(float(x) for x in clip) != (-1.0, 1.0):
                raise NotImplementedError(f"{name}: clip {clip} (the kernel clips the last action to +-1)")
        elif clip is not None:
            lo, hi = (float(x) for x in clip)
            if blind or lo != -hi:
                raise NotImplementedError(f"{name}: clip {clip} is not implemented for this observation group")
            c.obs_clip = hi
        if getattr(t, "scale", None) not in (None, 1, 1.0):
            raise NotImplementedError(f"{name}: observation scale")
        if blind and k < 4:
            n = getattr(t, "noise", None)
            std = 0.0
            if n is not None:
                if type(n).__name__ not in ("AdditiveGaussianNoiseCfg", "GaussianNoiseCfg") or float(getattr(n, "mean", 0.0)) != 0.0:
                    raise NotImplementedError(f"{name}: only zero-mean additive Gaussian noise is implemented")
                std = float(n.std)
            c.noise_std[k] = std


def _lower_rows(cfg, spec: T.TaskSpec, c, expected, task: str, device_terms: bool):
    """``cfg.observations.policy`` of the Elevation / Visual task.  Without ``device_terms``, or when the term list is not
    the built-in row's, it is validated onto the built-in row as before (a modified term list raises, naming the task).  With
    ``device_terms`` a group of the row's own terms whose effective noise (a noise with enable_corruption), clips or scales
    differ from the built-in row's is lowered to ``spec.row_terms`` (row_terms.py, wl_set_row_terms), refusing by term name
    what the kernels do not do; a group the built-in row restates exactly is validated as before."""
    group = cfg.observations.policy
    terms = [(k, t) for k, t in _fields(group) if hasattr(t, "func")]
    if not device_terms or [_fname(t) for _, t in terms] != expected or getattr(group, "concatenate_terms", True) is not True:
        _validate_obs(cfg, expected, c, task=task)
        return
    from . import row_terms
    kind = task.lower()
    corrupt = bool(getattr(group, "enable_corruption", False))
    table = []
    for k, (name, t) in enumerate(terms):
        if kind == "visual" and k == 0:                     # the camera term: its own augmentation, nothing of this path
            if getattr(t, "clip", None) is not None or getattr(t, "scale", None) not in (None, 1, 1.0) or (corrupt and getattr(t, "noise", None) is not None):
                raise NotImplementedError(f"{name}: noise, clip or scale on the camera term is not implemented")
            continue
        table.append((name,) + row_terms.lower_term(name, t.func, getattr(t, "noise", None) if corrupt else None, getattr(t, "clip", None),
                                                    getattr(t, "scale", None), getattr(t, "modifiers", None), getattr(t, "history_length", 0)))
    if row_terms.is_builtin(kind, [t[1:] for t in table]) and not getattr(group, "history_length", None):
        _validate_obs(cfg, expected, c, task=task)
        return
    if getattr(group, "history_length", None):
        raise NotImplementedError("policy observation group: history_length is not implemented")
    spec.row_terms = table


def _lower_critic(cfg, spec: T.TaskSpec, kind: str, group_name: str = "critic"):
    """``cfg.observations.critic`` (an ObservationGroupCfg next to ``policy``) -> ``spec.critic_terms``, the term table of
    ``wl_critic_observe``.  Anything the kernels do not do raises NotImplementedError naming the term; no group, no table."""
    group = getattr(cfg.observations, group_name, None)
    if group is None:
        return
    from . import privileged
    if kind != "drift":
        raise NotImplementedError(f"a {group_name} observation group on the {kind.capitalize()} task is not implemented "
                                  "(the asymmetric actor-critic covers the Drift family)")
    if getattr(group, "concatenate_terms", True) is not True:
        raise NotImplementedError(f"{group_name} observation group: concatenate_terms=False is not implemented")
    table = []
    for name, t in _fields(group):
        if not hasattr(t, "func"):
            continue
        noise = getattr(t, "noise", None) if getattr(group, "enable_corruption", False) or getattr(t, "noise", None) is not None else None
        fn, clip = privileged.lower_term(name, t.func, getattr(t, "params", None), getattr(t, "clip", None), noise, getattr(t, "scale", None))
        table.append((name, fn, clip))
    if not table:
        raise NotImplementedError(f"{group_name} observation group: no terms")
    privileged.check_width([(fn, c) for _, fn, c in table], f"{group_name} observation group " + ", ".join(n for n, _, _ in table))
    setattr(spec, "critic_terms" if group_name == "critic" else "teacher_terms", table)


def _lower_row_critic(cfg, spec: T.TaskSpec, group_name: str = "critic"):
    """An Elevation ``cfg.observations.critic`` (``device_terms=True`` only) -> ``spec.row_critic``: the policy row's six
    terms in row order, noise-free with their own clips and scales, then terms of the critic library (DESIGN 6s).  Anything
    else raises NotImplementedError naming the term: noise, history or modifiers, a per-element map scale, a map without a
    clip, row terms out of order, a term after them outside the library; a group that does not open with the row terms
    keeps the library path's refusal on Elevation."""
    group = getattr(cfg.observations, group_name, None)
    if group is None:
        return
    from . import privileged, row_terms
    if getattr(group, "concatenate_terms", True) is not True:
        raise NotImplementedError(f"{group_name} observation group: concatenate_terms=False is not implemented")
    terms = [(name, t) for name, t in _fields(group) if hasattr(t, "func")]
    head = row_terms.task_terms("elevation")
    fns = [_fname(t) for _, t in terms]
    if not fns or fns[0] not in head:
        _lower_critic(cfg, None, "elevation", group_name)   # a library-only group: refused as before
    for k, ((name, t), fn) in enumerate(zip(terms, fns)):
        if k < len(head) and fn != head[k]:
            raise NotImplementedError(f"{group_name} term {name}: {fn} at position {k}; a row critic opens with the Elevation row's "
                                      f"terms {list(head)} in row order")
    if len(terms) < len(head):
        raise NotImplementedError(f"{group_name} observation group {[n for n, _ in terms]}: a row critic opens with all six row terms {list(head)}")
    out, lib = [], []
    for k, (name, t) in enumerate(terms):
        nz = getattr(t, "noise", None)
        if k < len(head):
            row_terms.lower_critic_term(name, t.func, nz, getattr(t, "clip", None), getattr(t, "scale", None),
                                        getattr(t, "modifiers", None), getattr(t, "history_length", 0))
            params = {k2: v for k2, v in (("clip", getattr(t, "clip", None)), ("scale", getattr(t, "scale", None))) if v is not None}
            out.append((name, fns[k], params))
        else:
            if getattr(t, "modifiers", None) or getattr(t, "history_length", 0):
                raise NotImplementedError(f"{group_name} term {name}: history_length / modifiers are not implemented")
            fn, clip = privileged.lower_term(name, t.func, getattr(t, "params", None), getattr(t, "clip", None), nz, getattr(t, "scale", None))
            lib.append((fn, clip))
            out.append((name, fn, {"clip": (-clip, clip)} if clip else {}))
    privileged.check_width(lib, f"{group_name} observation group " + ", ".join(n for n, _ in terms[len(head):]))
    setattr(spec, "row_critic" if group_name == "critic" else "row_teacher", out)


def _lower_policy(cfg, spec: T.TaskSpec, c, device_terms: bool):
    """``cfg.observations.policy`` of the Drift family: BlindObsCfg's group is validated onto the built-in row as before;
    with ``device_terms`` any other group is lowered to ``spec.policy_terms``, the term table of ``wl_policy_observe``
    (policy_obs.py), refusing by term name what the kernel does not do.  Without the flag a modified group raises."""
    saved = (list(c.noise_std), c.obs_clip)
    try:
        _validate_obs(cfg, _OBS_BLIND, c, blind=True)
        return
    except NotImplementedError:
        if not device_terms:
            raise
    c.noise_std[:], c.obs_clip = saved                      # the built-in row keeps the task's defaults
    from . import policy_obs
    group = cfg.observations.policy
    if getattr(group, "concatenate_terms", True) is not True:
        raise NotImplementedError("policy observation group: concatenate_terms=False is not implemented")
    if getattr(group, "history_length", None):
        raise NotImplementedError("policy observation group: history_length is not implemented")
    table = []
    for name, t in _fields(group):
        if not hasattr(t, "func"):
            continue
        if getattr(t, "history_length", 0):
            raise NotImplementedError(f"policy term {name}: history_length is not implemented")
        table.append((name,) + policy_obs.lower_term(name, t.func, getattr(t, "params", None), getattr(t, "noise", None),
                                                     getattr(t, "clip", None), getattr(t, "scale", None), getattr(t, "modifiers", None)))
    if not table:
        raise NotImplementedError("policy observation group: no terms")
    policy_obs.check_width([t[1:] for t in table], "policy observation group " + ", ".join(t[0] for t in table))
    spec.policy_terms = table


def _lower_common(cfg, spec: T.TaskSpec):
    c = spec.cfg
    sim_dt, dec = float(cfg.sim.dt), int(cfg.decimation)
    c.sim_dt, c.decimation = sim_dt, dec
    c.substeps = max(1, math.ceil(sim_dt / 0.005 - 1e-9))
    spec.episode_length_s = float(cfg.episode_length_s)
    c.episode_length_s = spec.episode_length_s
    c.max_episode_length = math.ceil(spec.episode_length_s / (sim_dt * dec))
    # action term (exactly one in every registered task: actions.throttle_steer)
    terms = _fields(cfg.actions)
    if len(terms) != 1:
        raise NotImplementedError(f"expected one action term, got {[k for k, _ in terms]}")
    a = terms[0][1]
    kind = a.class_type.__name__
    if kind not in _ACTION_KINDS:
        raise NotImplementedError(f"action term {kind} is not implemented by the fused step")
    c.action_kind = _ACTION_KINDS[kind]
    if a.bounding_strategy not in _BOUND:
        raise NotImplementedError(f"bounding_strategy {a.bounding_strategy!r}")
    c.bounding = _BOUND[a.bounding_strategy]
    c.no_reverse = 1 if a.no_reverse else 0
    c.act_scale[0], c.act_scale[1] = a.scale
    c.act_offset[0], c.act_offset[1] = a.offset
    c.base_length, c.base_width, c.wheel_radius_cfg = a.base_length, a.base_width, a.wheel_radius
    pol = cfg.observations.policy
    c.enable_corruption = 1 if getattr(pol, "enable_corruption", False) else 0
    if getattr(cfg, "terminations", None) is None:         # play cfgs ("no terminations"): nothing ever ends an episode
        c.term_enable = 0
        spec.termination_names = []
    # curriculum
    spec.curriculum = []
    for name, term in _fields(getattr(cfg, "curriculum", None)):
        if _fname(term) != "increase_reward_weight_over_time":
            raise NotImplementedError(f"curriculum term {name}: {_fname(term)}")
        p = term.params
        spec.curriculum.append(T.CurriculumTerm(name, p["reward_term_name"], float(p["increase"]),
                                                int(p.get("episodes_per_increase", 1)), p.get("max_increases", math.inf)))
    spec._curriculum_dirty = True


def _device_term(spec, name, term, kind, device_terms) -> bool:
    """With ``device_terms``, a term whose function is in the device-term library (by module AND name, before any
    match by name against the built-in slots) joins ``spec.device_terms``; returns whether it did."""
    from . import device_terms as dtm
    if not device_terms or dtm.lookup(term.func) is None:
        return False
    if kind == "reward":
        spec.device_terms.append((name, term.func, "reward", float(term.weight), dict(term.params or {})))
    else:
        spec.device_terms.append((name, term.func, "time_out" if getattr(term, "time_out", False) else "termination", 0.0,
                                  dict(term.params or {})))
    return True


def _lower_rewards(cfg, spec, table, handlers, allow_python_terms=False, device_terms=False):
    c = spec.cfg
    names = [None] * len(table)
    for k in range(T_MAX := 8):
        c.rew_weight[k] = 0.0
    for name, term in _fields(getattr(cfg, "rewards", None)):
        if _device_term(spec, name, term, "reward", device_terms):
            continue
        fn = _ALIASES.get(_fname(term), _fname(term))
        if fn not in table:
            if allow_python_terms:      # the reference's own Python function, evaluated between the two halves of the staged step
                spec.python_reward_terms.append((name, term.func, float(term.weight), dict(term.params or {})))
                continue
            raise NotImplementedError(f"reward term {name} -> {fn} is not implemented by the fused step "
                                      f"(pass allow_python_terms=True to run it as a host-side term)")
        slot = table[fn]
        names[slot] = name
        c.rew_weight[slot] = float(term.weight)
        handlers.get(fn, lambda p: None)(term.params or {})
    if any(n is None for n in names):
        missing = [f for f, s in table.items() if names[s] is None]
        # absent terms keep weight 0 (skipped by the reward manager); give them placeholder names
        for f in missing:
            names[table[f]] = f
    spec.reward_names = names
    c.num_rew_terms = len(names)
    T.set_curriculum(c, names, spec.curriculum)     # reward slots are known now


def _event_mode(name, term) -> bool:
    """Whether a DR event term is in IsaacLab's reset mode (True) or start-up mode (False); anything else is refused by name."""
    mode = getattr(term, "mode", "startup")
    if mode not in ("startup", "reset"):
        raise NotImplementedError(f"event term {name}: mode {mode!r} (the DR events are implemented in 'startup' and 'reset' mode)")
    if int(getattr(term, "min_step_count_between_reset", 0) or 0) != 0:
        raise NotImplementedError(f"event term {name}: min_step_count_between_reset "
                                  f"{term.min_step_count_between_reset} (only the default 0 is implemented)")
    return mode == "reset"


EVENT_MODES = ("startup", "reset", "interval")
MAX_INTERVAL_EVENTS = 8             # WL_MAX_EVENT_TERMS: the interval timers of one handle


def check_event_term(name, mode, interval_range_s=None, is_global_time=False, min_step_count_between_reset=0):
    """The refusals of a host-side (Python) event term, by name (env.add_event_term and the lowering of a cfg's event term)."""
    if mode not in EVENT_MODES:
        raise NotImplementedError(f"event term {name}: mode {mode!r} (Python event terms run in 'startup', 'reset' and 'interval' mode)")
    if is_global_time:
        raise NotImplementedError(f"event term {name}: is_global_time=True (the interval timers are per env and restart at reset)")
    if int(min_step_count_between_reset or 0) != 0:
        raise NotImplementedError(f"event term {name}: min_step_count_between_reset {min_step_count_between_reset} "
                                  "(only the default 0 is implemented)")
    if mode == "interval":
        if interval_range_s is None:
            raise ValueError(f"event term {name}: an interval event needs interval_range_s")
        lo, hi = (float(v) for v in interval_range_s)
        if not (math.isfinite(lo) and math.isfinite(hi) and 0.0 <= lo <= hi):
            raise ValueError(f"event term {name}: interval_range_s {tuple(interval_range_s)} must be finite with 0 <= lo <= hi")


def _python_event(spec, name, term, fn, allow_python_terms):
    """An event term whose function the kernels do not lower: a host-side event term of the spec (spec.python_event_terms,
    in cfg order) with ``allow_python_terms``, else refused by name."""
    if not allow_python_terms:
        raise NotImplementedError(f"event term {name} -> {fn}")
    mode = getattr(term, "mode", "startup")
    rng = getattr(term, "interval_range_s", None)
    check_event_term(name, mode, rng, bool(getattr(term, "is_global_time", False)), getattr(term, "min_step_count_between_reset", 0))
    if mode == "interval" and sum(1 for e in spec.python_event_terms if e[2] == "interval") >= MAX_INTERVAL_EVENTS:
        raise NotImplementedError(f"event term {name}: more than {MAX_INTERVAL_EVENTS} Python interval event terms")
    spec.python_event_terms.append((name, term.func, mode, dict(term.params or {}), tuple(float(v) for v in rng) if mode == "interval" else None))


def _device_event(spec, name, term, device_terms) -> bool:
    """With ``device_terms``, an event term whose function is in the device event library (device_events.REGISTRY) becomes
    a device event term of the spec (spec.device_events, in cfg order), after check_event_term's refusals and the
    library's own; returns whether it did."""
    from . import device_events as dev
    if not device_terms or dev.lookup(term.func) is None:
        return False
    mode = getattr(term, "mode", "startup")
    rng = getattr(term, "interval_range_s", None)
    check_event_term(name, mode, rng, bool(getattr(term, "is_global_time", False)), getattr(term, "min_step_count_between_reset", 0))
    dev.check_mode(name, mode)
    if len(spec.device_events) >= dev.MAX_TERMS:
        raise NotImplementedError(f"event term {name}: more than {dev.MAX_TERMS} device event terms")
    dev.velocity_ranges(name, term.params)
    spec.device_events.append((name, term.func, mode, dict(term.params or {}), tuple(float(v) for v in rng) if mode == "interval" else None))
    return True


def _lower_material_and_mass_events(events, spec, seed):
    """DR events shared by the tasks (randomize_rigid_body_material / _mass, randomize_actuator_gains): their ranges into the
    config; those in mode="reset" into ``spec.reset_events`` (redrawn at every reset, wl_set_reset_events)."""
    c = spec.cfg
    wheel_mass = None
    reset = []
    for name, term in events.items():
        fn, p = _fname(term), (term.params or {})
        if fn not in ("randomize_rigid_body_material", "randomize_actuator_gains", "randomize_rigid_body_mass"):
            continue
        if _event_mode(name, term):
            bodies = getattr(p.get("asset_cfg"), "body_names", None)
            reset.append({"randomize_rigid_body_material": "material", "randomize_actuator_gains": "actuator_gains"}.get(
                fn, "wheel_mass" if bodies is not None and "wheel" in str(bodies) else "base_mass"))
        if fn == "randomize_rigid_body_material":
            c.dr_num_buckets = int(p["num_buckets"])
            D, Cs = T.material_buckets(c.dr_num_buckets, p["static_friction_range"], p["dynamic_friction_range"],
                                       p.get("make_consistent", False), c.ground_mu_s, c.ground_mu_d, seed)
            for k in range(c.dr_num_buckets):
                c.dr_bucket_D[k], c.dr_bucket_C[k] = D[k], Cs[k]
        elif fn == "randomize_actuator_gains":
            c.dr_kd_range[0], c.dr_kd_range[1] = p["damping_distribution_params"]
        elif fn == "randomize_rigid_body_mass":
            bodies = getattr(p["asset_cfg"], "body_names", None)
            op = p.get("operation", "add")
            if bodies is not None and "wheel" in str(bodies):
                if op != "abs":
                    raise NotImplementedError(f"{name}: wheel mass randomisation with operation {op!r}")
                wheel_mass = p["mass_distribution_params"]
            else:
                c.dr_mass_add[0], c.dr_mass_add[1] = p["mass_distribution_params"]
                c.dr_mass_mode = {"add": 0, "abs": 1}[op]
    c.dr_wheel_mass_enable = 1 if wheel_mass is not None else 0
    if wheel_mass is not None:
        c.dr_wheel_mass[0], c.dr_wheel_mass[1] = wheel_mass
    spec.reset_events = [e for e in _RESET_EVENTS if e in reset]


def spec_from_reference_cfg(cfg, env_id_offset: int = 0, allow_python_terms: bool = False, device_terms: bool = False) -> T.TaskSpec:
    """Build the TaskSpec for a reference env-cfg instance: the train cfgs of the four registered ids (Drift, F1Tenth drift,
    Elevation, Visual, incl. MushrVisualRLRandomEnvCfg) and their play cfgs (rewards / terminations / curriculum = None).
    With ``allow_python_terms`` reward / termination terms the kernels do not implement are kept as host-side terms that
    call the cfg's own function (staged step, env.add_reward_term); otherwise they raise.  With ``device_terms`` such a
    term whose function is in the device-term library (device_terms.REGISTRY) becomes a device term of the spec
    (spec.device_terms, in cfg order, with the cfg's weight and params), matched by module and name before the
    built-in terms are matched by name.  With ``allow_python_terms`` an event term whose function the kernels do not lower
    becomes a host-side event term (spec.python_event_terms, registered by the env with add_event_term) in startup, reset or
    interval mode; the built-in event functions keep their own refusals.  With ``device_terms`` an Elevation or Visual event
    term whose function is in the device event library (IsaacLab's push_by_setting_velocity) becomes a device event term
    (spec.device_events, applied by wl_step_terms); the Drift family keeps lowering it onto its two built-in push slots."""
    num_envs = int(cfg.scene.num_envs)
    seed = int(cfg.seed) if getattr(cfg, "seed", None) is not None else 42
    kind = _task_kind(cfg)
    if getattr(cfg.observations, "critic", None) is not None and kind != "drift" and not (kind == "elevation" and device_terms):
        _lower_critic(cfg, None, kind)                      # (refused by name before anything is lowered)
    if device_terms and getattr(cfg.observations, "teacher", None) is not None:
        if getattr(cfg.observations, "critic", None) is not None:
            raise NotImplementedError("an env has a critic observation group or a teacher observation group, not both")
        if kind == "visual":
            _lower_critic(cfg, None, kind, "teacher")       # (refused by name, as a Visual critic group)
    if kind == "visual":
        return _lower_visual(cfg, num_envs, seed, env_id_offset, allow_python_terms, device_terms)
    if kind == "drift":
        events = dict(_fields(cfg.events))
        randomize = "change_wheel_friction" in events
        drive = "4wd" if cfg.actions.throttle_steer.class_type.__name__ != "RCCarRWDAction" else "2wd"
        usd = str(getattr(getattr(cfg.scene.robot, "spawn", None), "usd_path", "")).lower()
        spec = T.drift_task(num_envs=num_envs, seed=seed, env_id_offset=env_id_offset, randomize=randomize, drive=drive,
                            vehicle="f1tenth" if "f1tenth" in usd else "mushr")
        c = spec.cfg
        _lower_common(cfg, spec)
        _lower_policy(cfg, spec, c, device_terms)
        _lower_critic(cfg, spec, kind)
        if device_terms:
            _lower_critic(cfg, spec, kind, "teacher")

        def h_slip(p):
            c.slip_min_thresh, c.slip_max_thresh = p["min_thresh"], p["max_thresh"]
            c.slip_min_vel_x = p.get("min_vel_x", 0.5)

        def h_vel(p):
            c.vel_speed_target = p.get("speed_target", T.MAX_SPEED)
            c.vel_offset = p.get("offset", -T.MAX_SPEED ** 2)

        def h_ctd(p):
            c.trk_straight = p["straight"]
            c.ctd_track_radius = p.get("track_radius", (T.CORNER_IN_RADIUS + T.CORNER_OUT_RADIUS) / 2)
            c.ctd_offset = p.get("offset", -1.0)
            if p.get("p", 1.0) != 1:
                raise NotImplementedError("cross_track_dist with p != 1")

        _lower_rewards(cfg, spec, _DRIFT_REWARDS, {
            "side_slip": h_slip, "vel_dist": h_vel, "cross_track_dist": h_ctd,
            "turn_left_go_right": lambda p: setattr(c, "tlgr_ang_vel_thresh", p.get("ang_vel_thresh", math.pi / 4)),
            "energy_through_turn": lambda p: setattr(c, "energy_straight", p["straight"]),
        }, allow_python_terms, device_terms)
        for name, term in _fields(getattr(cfg, "terminations", None)):
            fn = _fname(term)
            if _device_term(spec, name, term, "termination", device_terms):
                continue
            if fn == "cart_off_track":
                p = term.params
                c.trk_straight, c.trk_corner_in, c.trk_corner_out = p["straight"], p["corner_in_radius"], p["corner_out_radius"]
            elif fn != "time_out":
                if not allow_python_terms:
                    raise NotImplementedError(f"termination term {name} -> {fn} (pass allow_python_terms=True to run it host-side)")
                spec.python_termination_terms.append((name, term.func, bool(getattr(term, "time_out", False)), dict(term.params or {})))
        for name, term in events.items():
            fn, p = _fname(term), term.params
            if fn == "reset_root_state_along_track":
                c.num_ref_poses = int(p.get("num_points", 20))
                c.reset_pos_noise, c.reset_yaw_noise = p.get("pos_noise", 0.0), p.get("yaw_noise", 0.0)
                poses = T.generate_reference_poses(c.num_ref_poses, p.get("track_radius", 0.8), p.get("track_straight_dist", 0.8), seed)
                for k, v in enumerate(poses.reshape(-1)):
                    c.ref_poses[k] = v
            elif fn in ("randomize_rigid_body_material", "randomize_actuator_gains", "randomize_rigid_body_mass"):
                pass                                            # lowered together below
            elif fn == "push_by_setting_velocity":
                vr = p["velocity_range"]
                if "x" in vr:                                   # high-frequency push
                    c.push_hf_interval[0], c.push_hf_interval[1] = term.interval_range_s
                    c.push_hf_range[0], c.push_hf_range[1], c.push_hf_range[2] = vr["x"][1], vr.get("y", (0, 0))[1], vr["yaw"][1]
                else:
                    c.push_lf_interval[0], c.push_lf_interval[1] = term.interval_range_s
                    c.push_lf_yaw = vr["yaw"][1]
            elif fn == "disable_all_lidars":
                pass                                            # no-op without omni.isaac.sensor (quirk Q15)
            else:
                _python_event(spec, name, term, fn, allow_python_terms)
        _lower_material_and_mass_events(events, spec, seed)
        return spec
    # elevation (elevation/mushr_elevation_env_cfg.py)
    spec = T.elevation_task(num_envs=num_envs, seed=seed, env_id_offset=env_id_offset)
    c = spec.cfg
    _lower_common(cfg, spec)
    _lower_rows(cfg, spec, c, _OBS_ELEV, "Elevation", device_terms)
    if device_terms:
        _lower_row_critic(cfg, spec)
        _lower_row_critic(cfg, spec, "teacher")
    for _, t in _fields(cfg.observations.policy):
        if hasattr(t, "func") and _fname(t) == "world_height_map":
            c.scan_offset, c.scan_plane_init = float(t.params["offset"]), float(t.params["plane_init_value"])
    _lower_rewards(cfg, spec, _ELEV_REWARDS, {}, allow_python_terms, device_terms)
    term_bits = {"time_out": 0, "root_height_below_minimum": 1, "stuck": 2, "upright_bool": 3, "close_to_goal": 4}
    if getattr(cfg, "terminations", None) is not None:
        mask = 0
        for name, term in _fields(cfg.terminations):
            fn, p = _fname(term), (term.params or {})
            if _device_term(spec, name, term, "termination", device_terms):
                continue
            if fn not in term_bits:
                if not allow_python_terms:
                    raise NotImplementedError(f"termination term {name} -> {fn} (pass allow_python_terms=True to run it host-side)")
                spec.python_termination_terms.append((name, term.func, bool(getattr(term, "time_out", False)), dict(p)))
                continue
            mask |= 1 << term_bits[fn]
            if fn == "root_height_below_minimum":
                c.elev_min_height = float(p["minimum_height"])
            elif fn == "stuck":
                c.elev_stuck_min_vel, c.elev_stuck_spin = float(p.get("min_vel", c.elev_stuck_min_vel)), float(p.get("spin_thresh", c.elev_stuck_spin))
            elif fn == "close_to_goal":
                c.elev_goal_dist = float(p.get("threshold", p.get("dist", c.elev_goal_dist)))
        c.term_enable = mask
    events = dict(_fields(cfg.events))
    for name, term in events.items():
        fn, p = _fname(term), (term.params or {})
        if fn == "reset_root_state_uniform":
            pr, vr = p["pose_range"], p.get("velocity_range", {})
            c.elev_reset_xy[0], c.elev_reset_xy[1] = pr["x"]
            c.elev_reset_yaw = float(pr["yaw"][1])
            if "x" in vr:
                c.elev_reset_vel[0], c.elev_reset_vel[1] = vr["x"]
        elif fn not in ("randomize_rigid_body_material", "randomize_actuator_gains", "randomize_rigid_body_mass") and \
                not _device_event(spec, name, term, device_terms):
            _python_event(spec, name, term, fn, allow_python_terms)
    _lower_material_and_mass_events(events, spec, seed)
    cmds = dict(_fields(getattr(cfg, "commands", None)))
    for name, term in cmds.items():
        rng = getattr(term, "ranges", None)
        if rng is not None and hasattr(rng, "pos_x"):
            c.cmd_pos_range[0], c.cmd_pos_range[1] = rng.pos_x
        rt = getattr(term, "resampling_time_range", None)
        if rt is not None:
            c.cmd_resample_s = float(rt[0])
    return spec


def _lower_visual(cfg, num_envs, seed, env_id_offset, allow_python_terms, device_terms=False):
    """MushrVisualRLEnvCfg / MushrVisualRLRandomEnvCfg / MushrVisualPlayEnvCfg (visual/mushr_visual_env_cfg.py:412-473)."""
    import numpy as np
    terrain = cfg.scene.terrain
    trav = np.asarray(terrain.traversability_hashmap, dtype=bool)
    funcs = _obs_funcs(cfg)
    cam_mode = _CAMERA_FUNCS[funcs[0]]
    events = dict(_fields(cfg.events))
    randomize = "change_wheel_friction" in events
    spec = T.visual_task(num_envs=num_envs, seed=seed, env_id_offset=env_id_offset, traversability=trav, camera=cam_mode, randomize=randomize)
    c = spec.cfg
    _lower_common(cfg, spec)
    _lower_rows(cfg, spec, c, [funcs[0]] + _OBS_VIS_TAIL, "Visual", device_terms)
    # map geometry (VisualTerrainImporterCfg :63-124) and ground material (:126-135)
    c.vis_row_spacing, c.vis_col_spacing = float(terrain.row_spacing), float(terrain.col_spacing)
    c.vis_width, c.vis_height = float(terrain.width), float(terrain.height)
    c.vis_mesh_x0 = -c.vis_width / 2 - c.vis_row_spacing / 2
    c.vis_mesh_y0 = -c.vis_height / 2 - c.vis_col_spacing / 2
    c.vis_mesh_dx, c.vis_mesh_dy = c.vis_width / (c.vis_rows - 1), c.vis_height / (c.vis_cols - 1)
    mat = getattr(terrain, "physics_material", None)
    if mat is not None:
        if getattr(mat, "friction_combine_mode", "multiply") != "multiply":
            raise NotImplementedError("ground friction combine mode other than 'multiply'")
        c.ground_mu_s, c.ground_mu_d = float(mat.static_friction), float(mat.dynamic_friction)
    # camera (TiledCameraCfg :230-246)
    cam = cfg.scene.camera
    c.vis_cam_w, c.vis_cam_h = int(cam.width), int(cam.height)
    c.vis_cam_row0 = c.vis_cam_h // 3
    sp = cam.spawn
    c.vis_cam_fx = float(sp.focal_length) * c.vis_cam_w / float(sp.horizontal_aperture)
    c.vis_cam_fy = float(sp.focal_length) * c.vis_cam_h / float(sp.vertical_aperture)
    c.vis_cam_cx, c.vis_cam_cy = c.vis_cam_w / 2.0, c.vis_cam_h / 2.0
    off = cam.offset.pos
    c.vis_cam_pos[0], c.vis_cam_pos[1], c.vis_cam_pos[2] = 0.022995 + float(off[0]), 0.0175 + float(off[1]), 0.162178 + float(off[2])
    spec.obs_dim = 8 + c.vis_cam_w * (c.vis_cam_h - c.vis_cam_row0)
    _lower_rewards(cfg, spec, _VIS_REWARDS, {}, allow_python_terms, device_terms)
    if getattr(cfg, "terminations", None) is not None:
        mask = 0
        for name, term in _fields(cfg.terminations):
            fn = _fname(term)
            if _device_term(spec, name, term, "termination", device_terms):
                continue
            if fn == "time_out":
                mask |= 1
            elif fn == "out_of_map":
                mask |= 2
            elif allow_python_terms:
                spec.python_termination_terms.append((name, term.func, bool(getattr(term, "time_out", False)), dict(term.params or {})))
            else:
                raise NotImplementedError(f"termination term {name} -> {fn} (pass allow_python_terms=True to run it host-side)")
        c.term_enable = mask
    for name, term in events.items():
        fn = _fname(term)
        if fn not in ("reset_root_state", "randomize_rigid_body_material", "randomize_actuator_gains", "randomize_rigid_body_mass") and \
                not _device_event(spec, name, term, device_terms):
            _python_event(spec, name, term, fn, allow_python_terms)
    if randomize:
        _lower_material_and_mass_events(events, spec, seed)
    else:                                                      # material table follows the (possibly overridden) ground friction
        D, Cs = T.material_buckets(1, (1.0, 1.0), (1.0, 1.0), True, c.ground_mu_s, c.ground_mu_d, seed)
        c.dr_bucket_D[0], c.dr_bucket_C[0] = D[0], Cs[0]
    return spec


def env_from_reference_cfg(cfg, render_mode=None, device=None, allow_python_terms: bool = False, device_terms: bool = False, **kwargs):
    """Entry point used by ``shims/isaaclab/envs:ManagerBasedRLEnv`` (gym kwargs: cfg=<env cfg>)."""
    from .env import ManagerBasedRLEnv
    kwargs.pop("env_cfg_entry_point", None); kwargs.pop("rsl_rl_cfg_entry_point", None); kwargs.pop("play_env_cfg_entry_point", None)
    if isinstance(cfg, (str, T.TaskSpec)):           # a gym id / an already lowered TaskSpec instead of a reference cfg object
        return ManagerBasedRLEnv(cfg, render_mode=render_mode, device=device or "cuda:0")
    dev = device or getattr(getattr(cfg, "sim", None), "device", None) or "cuda:0"
    env = ManagerBasedRLEnv(spec_from_reference_cfg(cfg, allow_python_terms=allow_python_terms, device_terms=device_terms), render_mode=render_mode, device=dev)
    env.cfg = cfg                                   # writer.log_config(self.env.cfg, ...) (modified_rsl_rl_runner.py:42-44)
    if not hasattr(cfg, "is_finite_horizon"):
        cfg.is_finite_horizon = False
    return env
