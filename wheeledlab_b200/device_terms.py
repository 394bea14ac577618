"""Device terms: the reward / termination functions the reference's task files define without registering them, run by
a CUDA kernel between the two halves of the staged step (``wl_set_device_terms`` / ``wl_step_terms``, DESIGN.md 6l).

The registry maps a reference function, identified by its module AND its name, to the kernel's term kind: the
reference defines ``forward_vel`` in both the Elevation and the Visual task files with different bodies, and
``off_track`` / ``upright_bool`` / ``is_falling_penalty`` more than once, so a name alone does not identify a function.
"""
from __future__ import annotations

import math
from dataclasses import dataclass

ELEVATION = "wheeledlab_tasks.elevation.mushr_elevation_env_cfg"
VISUAL = "wheeledlab_tasks.visual.mushr_visual_env_cfg"

ROLE_REWARD, ROLE_TERMINATION, ROLE_TIME_OUT = 0, 1, 2       # WL_TERM_ROLE_*
MAX_TERMS = 8                                               # WL_MAX_DEVICE_TERMS


@dataclass(frozen=True)
class TermKind:
    kind: int                 # WL_TERM_*
    module: str
    name: str
    params: tuple = ()        # (parameter name, the reference's default or None when it has none)
    map_term: bool = False    # reads the traversability map: Visual task only

    @property
    def key(self):
        return (self.module, self.name)


_KINDS = [
    TermKind(1, ELEVATION, "forward_vel"),
    TermKind(2, ELEVATION, "forward_wheel_spin"),
    TermKind(3, ELEVATION, "change_in_elevation"),
    TermKind(4, ELEVATION, "ascending"),
    TermKind(5, ELEVATION, "steep_penalty", (("thresh_pitch", None),)),
    TermKind(6, ELEVATION, "elevation_continuity", (("threshold_elev", None),)),
    TermKind(7, ELEVATION, "yaw_change_onElev", (("threshold_yaw", None), ("threshold_z", None))),
    TermKind(8, ELEVATION, "upright_penalty", (("thresh_deg", None),)),
    TermKind(9, ELEVATION, "roll_on_elev", (("z_start", None), ("roll_rate_thresh", None))),
    TermKind(10, ELEVATION, "low_vel_penalty", (("min_vel", 0.1),)),
    TermKind(11, VISUAL, "is_traversable", map_term=True),
    TermKind(12, VISUAL, "is_traversable_speed_scaled", map_term=True),
    TermKind(13, VISUAL, "vel_rew_trav", (("speed_target_on_trav", 1.0), ("speed_target_on_non_trav", 2.0)), map_term=True),
    TermKind(14, VISUAL, "low_speed_penalty", (("low_speed_thresh", 0.3),)),
    TermKind(15, VISUAL, "off_track", (("straight", None), ("corner_out_radius", None))),
    TermKind(16, VISUAL, "bool_is_not_traversable", map_term=True),
    TermKind(17, VISUAL, "roll_over"),
]
REGISTRY = {k.key: k for k in _KINDS}


def _module_of(func) -> str:
    """The reference module a function object comes from, with the package path the reference imports it by (a file
    loaded under another module name is recognised by its package-relative tail)."""
    mod = getattr(func, "__module__", None) or ""
    for full in (ELEVATION, VISUAL):
        tail = full.split(".", 1)[1]          # elevation.mushr_elevation_env_cfg
        if mod == full or mod.endswith("." + tail) or mod == tail:
            return full
    return mod


def lookup(func) -> TermKind | None:
    """The library entry of a reference function object, or None (a lambda, a function of another module, or one the
    library does not have)."""
    name = getattr(func, "__name__", None)
    if not name or name == "<lambda>":
        return None
    return REGISTRY.get((_module_of(func), name))


def resolve(kind: TermKind | int | str, module: str | None = None) -> TermKind:
    """A TermKind from itself, its WL_TERM_* number, or (module, name)."""
    if isinstance(kind, TermKind):
        return kind
    if isinstance(kind, int):
        for k in _KINDS:
            if k.kind == kind:
                return k
        raise ValueError(f"unknown device term kind {kind}")
    try:
        return REGISTRY[(module, kind)]
    except KeyError:
        raise ValueError(f"no device term {module}.{kind}") from None


def param_values(tk: TermKind, params: dict | None) -> list:
    """The term's parameters in kernel order (four doubles), from the cfg's params and the reference's defaults."""
    params = dict(params or {})
    unknown = set(params) - {n for n, _ in tk.params}
    if unknown:
        raise TypeError(f"{tk.name}() got unexpected parameters {sorted(unknown)}")
    vals = []
    for n, default in tk.params:
        v = params.get(n, default)
        if v is None:
            raise TypeError(f"{tk.name}() missing parameter {n!r}")
        v = float(v)
        if not math.isfinite(v):
            raise ValueError(f"{tk.name}: parameter {n} must be finite")
        vals.append(v)
    return vals + [0.0] * (4 - len(vals))
