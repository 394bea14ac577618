"""A modified policy observation group of the Drift family (DESIGN 6q): the term table of ``wl_policy_observe``.

A term is matched by the IsaacLab / reference function name (``root_pos_w``, ``root_euler_xyz``, ``base_lin_vel``,
``base_ang_vel``, ``last_action``, ``joint_vel``, ``joint_pos``, ``projected_gravity``) or is one of this project's
``privileged.wheel_friction`` / ``base_mass`` / ``motor_damping``.  Each term carries what IsaacLab's ObservationManager
applies after the value: additive noise (``AdditiveGaussianNoiseCfg`` / ``AdditiveUniformNoiseCfg``, drawn only when the
config's ``enable_corruption`` is set), a clip ``(lo, hi)`` and a scale (a number, or one per float).  A lowered term is
``(library name, noise, clip, scale)`` with noise ``None``, ``("gaussian", mean, std)`` or ``("uniform", n_min, n_max)``."""
from __future__ import annotations

import math

from ._lib import WL_POLICY_TERMS, WL_MAX_POLICY_OBS
from .privileged import _JOINTS


def _noise(name: str, noise):
    if noise is None:
        return None
    if isinstance(noise, tuple):
        return noise
    kind = type(noise).__name__
    if getattr(noise, "operation", "add") != "add":
        raise NotImplementedError(f"policy term {name}: noise operation {noise.operation!r} (only \"add\" is implemented)")
    if kind in ("AdditiveGaussianNoiseCfg", "GaussianNoiseCfg"):
        return ("gaussian", float(getattr(noise, "mean", 0.0)), float(getattr(noise, "std", 1.0)))
    if kind in ("AdditiveUniformNoiseCfg", "UniformNoiseCfg"):
        return ("uniform", float(getattr(noise, "n_min", -1.0)), float(getattr(noise, "n_max", 1.0)))
    raise NotImplementedError(f"policy term {name}: noise model {kind} (additive Gaussian and uniform noise are implemented)")


def lower_term(name: str, func, params: dict | None = None, noise=None, clip=None, scale=None, modifiers=None) -> tuple:
    """One term of a policy group -> ``(library name, noise, clip, scale)`` for ``sim.set_policy_terms``.  `func` is a library
    name or a function whose ``__name__`` is one.  Raises NotImplementedError, naming the term, for what the kernel does not
    do: a function outside the library, a noise model other than additive Gaussian / uniform, modifiers, joints other than
    the term's own; ValueError for a non-finite parameter or a scale of the wrong length."""
    fn = func if isinstance(func, str) else getattr(func, "__name__", type(func).__name__)
    if fn not in WL_POLICY_TERMS:
        raise NotImplementedError(f"policy term {name}: {fn} is not in the policy observation library {sorted(WL_POLICY_TERMS)}")
    if modifiers:
        raise NotImplementedError(f"policy term {name}: observation modifiers are not implemented")
    asset = (params or {}).get("asset_cfg")
    joints = getattr(asset, "joint_names", None)
    if fn in _JOINTS and joints is not None and not all(_JOINTS[fn] in str(j) for j in ([joints] if isinstance(joints, str) else joints)):
        raise NotImplementedError(f"policy term {name}: {fn} is implemented for the {_JOINTS[fn]} joints only, not {joints}")
    nz = _noise(name, noise)
    cl = None if clip is None else tuple(float(x) for x in clip)
    width = WL_POLICY_TERMS[fn][1]
    sc = None
    if scale is not None:
        sc = (float(scale),) if isinstance(scale, (int, float)) else tuple(float(x) for x in scale)
        if len(sc) not in (1, width):
            raise ValueError(f"policy term {name}: scale {scale} must be one number or {width} (the term's width)")
    vals = list(nz[1:] if nz else ()) + list(cl or ()) + list(sc or ())
    if not all(math.isfinite(v) for v in vals):
        raise ValueError(f"policy term {name}: a noise, clip or scale parameter is not finite")
    return fn, nz, cl, sc


def row_width(table) -> int:
    return sum(WL_POLICY_TERMS[t[0]][1] for t in table)


def check_width(table, name="policy group") -> int:
    dp = row_width(table)
    if dp > WL_MAX_POLICY_OBS:
        raise NotImplementedError(f"{name}: the policy row is {dp} floats wide, more than the {WL_MAX_POLICY_OBS} the kernels take")
    return dp


def blind_table(noise_std) -> list:
    """BlindObsCfg's five terms as a table: the built-in row of a handle with these observation noise stds."""
    names = ("root_pos_w", "root_euler_xyz", "base_lin_vel", "base_ang_vel")
    return [(n, ("gaussian", 0.0, float(s)), None, None) for n, s in zip(names, noise_std)] + [("last_action", None, (-1.0, 1.0), None)]
