"""Device event terms: IsaacLab event functions run by a CUDA kernel inside the step, in reset and interval mode
(``wl_set_device_events`` / ``wl_step_terms``, DESIGN.md 6p).

The library maps an event function, identified by its module AND its name as ``device_terms.REGISTRY`` identifies a
term, to what the kernel runs.  It has one entry, IsaacLab's ``push_by_setting_velocity`` [UPSTREAM-RECALL]: per fired
env, ``root_vel_w += U(lo, hi)`` per component of ``velocity_range`` (x, y, z, roll, pitch, yaw; a component it does not
name gets (0, 0)), written back with ``write_root_velocity_to_sim``.
"""
from __future__ import annotations

import math
from dataclasses import dataclass

ISAACLAB_MDP = "isaaclab.envs.mdp"
MODES = ("reset", "interval")
MAX_TERMS = 8                                               # WL_MAX_DEVICE_EVENTS
COMPONENTS = ("x", "y", "z", "roll", "pitch", "yaw")        # the order of wl_device_event_desc.velocity_range


@dataclass(frozen=True)
class EventKind:
    module: str
    name: str

    @property
    def key(self):
        return (self.module, self.name)


PUSH_BY_SETTING_VELOCITY = EventKind(ISAACLAB_MDP, "push_by_setting_velocity")
REGISTRY = {k.key: k for k in (PUSH_BY_SETTING_VELOCITY,)}


def _module_of(func) -> str:
    """``isaaclab.envs.mdp`` for a function of that package or one of its modules (IsaacLab defines the event functions in
    ``isaaclab.envs.mdp.events`` and re-exports them from the package)."""
    mod = getattr(func, "__module__", None) or ""
    return ISAACLAB_MDP if mod == ISAACLAB_MDP or mod.startswith(ISAACLAB_MDP + ".") else mod


def lookup(func) -> EventKind | None:
    """The library entry of an event function object, or None (a lambda, a function of another module, or one the library
    does not have)."""
    name = getattr(func, "__name__", None)
    if not name or name == "<lambda>":
        return None
    return REGISTRY.get((_module_of(func), name))


def check_mode(name: str, mode: str):
    """The refusal a device event term adds to compat.check_event_term's: startup mode."""
    if mode not in MODES:
        raise NotImplementedError(f"event term {name}: mode {mode!r} (device event terms run in 'reset' and 'interval' mode; a "
                                  "startup push is overwritten by the first reset)")


def velocity_ranges(name: str, params: dict | None) -> list:
    """push_by_setting_velocity's params as the kernel's six (lo, hi) pairs.  Refused by term name: a parameter the
    function does not take, a component it does not know, an asset other than ``robot``, a bound that is not finite or
    lo > hi."""
    params = dict(params or {})
    unknown = set(params) - {"velocity_range", "asset_cfg"}
    if unknown:
        raise TypeError(f"event term {name}: push_by_setting_velocity() got unexpected parameters {sorted(unknown)}")
    if "velocity_range" not in params:
        raise TypeError(f"event term {name}: push_by_setting_velocity() missing parameter 'velocity_range'")
    asset = params.get("asset_cfg")
    if asset is not None and getattr(asset, "name", "robot") != "robot":
        raise NotImplementedError(f"event term {name}: asset {getattr(asset, 'name', asset)!r} (the scene has one articulation, 'robot')")
    vr = dict(params["velocity_range"])
    bad = set(vr) - set(COMPONENTS)
    if bad:
        raise ValueError(f"event term {name}: velocity_range keys {sorted(bad)} (known: {', '.join(COMPONENTS)})")
    out = []
    for c in COMPONENTS:
        lo, hi = (float(v) for v in vr.get(c, (0.0, 0.0)))
        if not (math.isfinite(lo) and math.isfinite(hi) and lo <= hi):
            raise ValueError(f"event term {name}: velocity_range[{c!r}] {(lo, hi)} must be finite with lo <= hi")
        out.append((lo, hi))
    return out
