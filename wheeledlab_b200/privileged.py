"""The critic observation group of the Drift family (DESIGN 6m): the term library of ``wl_critic_observe`` as functions.

``wheel_friction``, ``base_mass`` and ``motor_damping`` are this project's own observation functions,
``fn(env, **params) -> tensor`` as IsaacLab's are, so a cfg's ``critic: ObservationGroupCfg`` can name them and a test can
call them as a Python restatement of the kernel's columns.  The other seven terms of the library are matched by the
IsaacLab / reference function names (``root_pos_w`` ... ``last_action``, ``joint_vel``, ``joint_pos``)."""
from __future__ import annotations

from ._lib import WL_CRITIC_TERMS, WL_MAX_CRITIC_OBS
from .sim import G_PKD, G_PMASS, G_PMU_D


def wheel_friction(env) -> "torch.Tensor":
    """[N, 4]: the peak friction coefficient of each wheel [bl, br, fl, fr], from the env's domain-randomisation bucket."""
    return env.sim.groups[G_PMU_D]


def base_mass(env) -> "torch.Tensor":
    """[N, 1]: the vehicle's total mass after the mass randomisation."""
    return env.sim.groups[G_PMASS, :, 0:1]


def motor_damping(env) -> "torch.Tensor":
    """[N, 4]: the DC-motor damping of each wheel after the actuator-gain randomisation."""
    return env.sim.groups[G_PKD]


_JOINTS = {"joint_vel": "throttle", "joint_pos": "steer"}


def lower_term(name: str, func, params: dict | None = None, clip=None, noise=None, scale=None) -> tuple:
    """One term of a critic group -> (library name, clip) for ``sim.set_critic_terms``.  `func` is a library name or a
    function whose ``__name__`` is one.  Raises NotImplementedError, naming the term, for what the kernel does not do:
    a function outside the library, noise, a scale, an asymmetric clip, joints other than the term's own."""
    fn = func if isinstance(func, str) else getattr(func, "__name__", type(func).__name__)
    if fn not in WL_CRITIC_TERMS:
        raise NotImplementedError(f"critic term {name}: {fn} is not in the critic observation library {sorted(WL_CRITIC_TERMS)}")
    if noise is not None:
        raise NotImplementedError(f"critic term {name}: noise on a critic term is not implemented (the critic row is noise-free)")
    if scale not in (None, 1, 1.0):
        raise NotImplementedError(f"critic term {name}: observation scale is not implemented")
    c = 0.0
    if clip is not None:
        lo, hi = (float(x) for x in clip)
        if lo != -hi or not hi > 0:
            raise NotImplementedError(f"critic term {name}: clip {clip} (only a symmetric clip is implemented)")
        c = hi
    asset = (params or {}).get("asset_cfg")
    joints = getattr(asset, "joint_names", None)
    if fn in _JOINTS and joints is not None and not all(_JOINTS[fn] in str(j) for j in ([joints] if isinstance(joints, str) else joints)):
        raise NotImplementedError(f"critic term {name}: {fn} is implemented for the {_JOINTS[fn]} joints only, not {joints}")
    return fn, c


def row_width(table) -> int:
    return sum(WL_CRITIC_TERMS[fn][1] for fn, _ in table)


def check_width(table, name="critic group") -> int:
    dc = row_width(table)
    if dc > WL_MAX_CRITIC_OBS:
        raise NotImplementedError(f"{name}: the critic row is {dc} floats wide, more than the {WL_MAX_CRITIC_OBS} the kernels take")
    return dc
