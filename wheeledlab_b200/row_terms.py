"""Noise, clip and scale on the Elevation and Visual policy rows (DESIGN 6r): the row terms of ``wl_set_row_terms``.

The row keeps the task's built-in terms in their order (``_lib.WL_ROW_TASK_TERMS``); each term carries what IsaacLab's
ObservationManager applies after the value: additive noise (``AdditiveGaussianNoiseCfg`` / ``AdditiveUniformNoiseCfg``,
drawn only when the config's ``enable_corruption`` is set), a clip ``(lo, hi)`` and a scale (a number, or one per float;
one number on the height map).  A lowered term is ``(row term name, noise, clip, scale)`` with noise ``None``,
``("gaussian", mean, std)`` or ``("uniform", n_min, n_max)``."""
from __future__ import annotations

import math

from ._lib import WL_ROW_TASK_TERMS, WL_ROW_TERMS
from .policy_obs import _noise


def task_terms(task: str) -> tuple:
    """The function names of the task's built-in row, in order ("elevation" / "visual")."""
    if task not in WL_ROW_TASK_TERMS:
        raise NotImplementedError(f"row terms are implemented for the Elevation and Visual tasks, not {task!r} "
                                  "(the Drift family's policy group goes through the policy observation table)")
    return WL_ROW_TASK_TERMS[task]


def lower_term(name: str, func, noise=None, clip=None, scale=None, modifiers=None, history_length=0) -> tuple:
    """One term of an Elevation / Visual policy group -> ``(row term, noise, clip, scale)`` for ``sim.set_row_terms``.  `func`
    is a row term's name or a function whose ``__name__`` is one.  Raises NotImplementedError, naming the term, for what the
    kernels do not do (a noise model other than additive Gaussian / uniform, an operation other than "add", modifiers,
    history_length, a per-element scale on the height map) and ValueError for a non-finite parameter or a scale of the
    wrong length."""
    fn = func if isinstance(func, str) else getattr(func, "__name__", type(func).__name__)
    if fn not in WL_ROW_TERMS:
        raise NotImplementedError(f"row term {name}: {fn} is not a term of the Elevation or Visual row")
    if modifiers:
        raise NotImplementedError(f"row term {name}: observation modifiers are not implemented")
    if history_length:
        raise NotImplementedError(f"row term {name}: history_length is not implemented")
    nz = _noise(name, noise)
    cl = None if clip is None else tuple(float(x) for x in clip)
    width = WL_ROW_TERMS[fn][1]
    sc = None
    if scale is not None:
        sc = (float(scale),) if isinstance(scale, (int, float)) else tuple(float(x) for x in scale)
        if fn == "world_height_map" and len(sc) != 1:
            raise NotImplementedError(f"row term {name}: a per-element scale on the height map is not implemented (one number)")
        if len(sc) not in (1, width):
            raise ValueError(f"row term {name}: scale {scale} must be one number or {width} (the term's width)")
    vals = list(nz[1:] if nz else ()) + list(cl or ()) + list(sc or ())
    if not all(math.isfinite(v) for v in vals):
        raise ValueError(f"row term {name}: a noise, clip or scale parameter is not finite")
    return fn, nz, cl, sc


def lower_critic_term(name: str, func, noise=None, clip=None, scale=None, modifiers=None, history_length=0) -> tuple:
    """``lower_term`` for one of the six row terms that open an Elevation row critic (DESIGN 6s): the critic row is
    noise-free, and a height map without a clip would hand a miss (+inf) to the critic, so both are refused by name."""
    if noise is not None:
        raise NotImplementedError(f"critic term {name}: noise on a critic term is not implemented (the critic row is noise-free)")
    t = lower_term(name, func, None, clip, scale, modifiers, history_length)
    if t[0] == "world_height_map" and t[2] is None:
        raise NotImplementedError(f"critic term {name}: the critic's height map needs a finite clip (a ray that misses is +inf)")
    return t


def check_order(task: str, fns) -> None:
    """Row terms name the row's own terms in its order: anything else is a modified term list, which is not implemented."""
    expected = task_terms(task)
    if tuple(fns) != expected:
        raise NotImplementedError(f"row terms {list(fns)} differ from the {task.capitalize()} row's {list(expected)} (order matters; "
                                  "a modified term list is not implemented)")


def registered(task: str, obs_clip: float = 10.0) -> list:
    """The row terms that restate the built-in row exactly, no noise and no scale: on Elevation one shared symmetric clip
    (+-obs_clip) on the two velocity terms and the map, +-1 on last_action, none on goal and euler; on Visual +-1 on
    last_action and no other clip."""
    vel = (-float(obs_clip), float(obs_clip)) if task == "elevation" else None
    clips = {"goal_relative_xyz": None, "root_euler_xyz": None, "base_lin_vel": vel, "base_ang_vel": vel,
             "last_action": (-1.0, 1.0), "world_height_map": vel}
    return [(fn, None, clips[fn], None) for fn in task_terms(task)]


def is_builtin(task: str, table) -> bool:
    """Whether lowered row terms are what the built-in row does exactly (so that the config's obs_clip expresses them)."""
    if any(nz is not None or sc is not None for _, nz, _, sc in table):
        return False
    clips = [cl for _, _, cl, _ in table]
    if task == "visual":
        return clips == [None, None, (-1.0, 1.0)]
    shared = clips[2]
    return (shared is not None and shared[0] == -shared[1] and clips[3] == shared and clips[5] == shared
            and clips[0] is None and clips[1] is None and clips[4] == (-1.0, 1.0))
