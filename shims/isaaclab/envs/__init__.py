"""isaaclab.envs stand-in.  ``ManagerBasedRLEnv`` resolves to the wheeledlab_b200 drop-in when it is
constructed (shims stay importable on a machine without the CUDA library for config-only use)."""
from dataclasses import MISSING

from ..sim import SimulationCfg
from ..utils import configclass
from . import mdp  # noqa: F401


@configclass
class ViewerCfg:
    eye: tuple = (7.5, 7.5, 7.5)
    lookat: tuple = (0.0, 0.0, 0.0)
    cam_prim_path: str = "/OmniverseKit_Persp"
    resolution: tuple = (1280, 720)
    origin_type: str = "world"
    env_index: int = 0
    asset_name: object = None
    body_name: object = None


@configclass
class ManagerBasedEnvCfg:
    viewer: ViewerCfg = ViewerCfg()
    sim: SimulationCfg = SimulationCfg()
    ui_window_class_type: object = None
    seed: object = None
    decimation: int = MISSING
    scene: object = MISSING
    recorders: object = None
    observations: object = MISSING
    actions: object = MISSING
    events: object = None
    rerender_on_reset: bool = False
    wait_for_textures: bool = True


@configclass
class ManagerBasedRLEnvCfg(ManagerBasedEnvCfg):
    is_finite_horizon: bool = False
    episode_length_s: float = MISSING
    rewards: object = MISSING
    terminations: object = MISSING
    curriculum: object = None
    commands: object = None


class _LazyEnvMeta(type):
    """isinstance(env, isaaclab.envs.ManagerBasedRLEnv) is true for the wheeledlab_b200 drop-in."""

    def __instancecheck__(cls, inst):
        try:
            from wheeledlab_b200.env import ManagerBasedRLEnv as _Real
        except Exception:
            return type.__instancecheck__(cls, inst)
        return isinstance(inst, _Real) or type.__instancecheck__(cls, inst)


class ManagerBasedEnv(metaclass=_LazyEnvMeta):
    pass


class ManagerBasedRLEnv(ManagerBasedEnv):
    """gym entry point 'isaaclab.envs:ManagerBasedRLEnv' (wheeledlab_tasks/__init__.py:16): construct the
    fused-step env from the reference's own cfg object."""

    def __new__(cls, cfg=None, render_mode=None, **kwargs):
        from wheeledlab_b200.compat import env_from_reference_cfg
        return env_from_reference_cfg(cfg, render_mode=render_mode, **kwargs)
