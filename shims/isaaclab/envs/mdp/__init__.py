"""isaaclab.envs.mdp stand-in: state accessors + term functions the reference's cfgs reference.
Accessors are [UPSTREAM-RECALL isaaclab/envs/mdp/{observations,terminations,rewards}.py]; event functions
are identity markers that wheeledlab_b200.compat lowers onto the kernels by ``__name__``."""
import torch

from ...managers import SceneEntityCfg
from ...utils.math import euler_xyz_from_quat  # noqa: F401  (reference: mdp.euler_xyz_from_quat)
from . import commands, events, rewards  # noqa: F401
from .commands import UniformPose2dCommandCfg  # noqa: F401
from .events import (push_by_setting_velocity, randomize_actuator_gains, randomize_rigid_body_mass,  # noqa: F401
                     randomize_rigid_body_material, reset_root_state_uniform, reset_scene_to_default)
from .rewards import is_terminated, is_terminated_term  # noqa: F401

_ROBOT = SceneEntityCfg("robot")


def root_pos_w(env, asset_cfg: SceneEntityCfg = _ROBOT):
    asset = env.scene[asset_cfg.name]
    return asset.data.root_pos_w - env.scene.env_origins


def root_quat_w(env, make_quat_unique: bool = False, asset_cfg: SceneEntityCfg = _ROBOT):
    return env.scene[asset_cfg.name].data.root_quat_w


def root_lin_vel_w(env, asset_cfg: SceneEntityCfg = _ROBOT):
    return env.scene[asset_cfg.name].data.root_lin_vel_w


def root_ang_vel_w(env, asset_cfg: SceneEntityCfg = _ROBOT):
    return env.scene[asset_cfg.name].data.root_ang_vel_w


def base_lin_vel(env, asset_cfg: SceneEntityCfg = _ROBOT):
    return env.scene[asset_cfg.name].data.root_lin_vel_b


def base_ang_vel(env, asset_cfg: SceneEntityCfg = _ROBOT):
    return env.scene[asset_cfg.name].data.root_ang_vel_b


def projected_gravity(env, asset_cfg: SceneEntityCfg = _ROBOT):
    return env.scene[asset_cfg.name].data.projected_gravity_b


def base_pos_z(env, asset_cfg: SceneEntityCfg = _ROBOT):
    return env.scene[asset_cfg.name].data.root_pos_w[:, 2].unsqueeze(-1)


def joint_pos(env, asset_cfg: SceneEntityCfg = _ROBOT):
    return env.scene[asset_cfg.name].data.joint_pos[:, asset_cfg.joint_ids]


def joint_vel(env, asset_cfg: SceneEntityCfg = _ROBOT):
    return env.scene[asset_cfg.name].data.joint_vel[:, asset_cfg.joint_ids]


def last_action(env, action_name=None):
    return env.action_manager.action


def generated_commands(env, command_name: str):
    return env.command_manager.get_command(command_name)


def height_scan(env, sensor_cfg: SceneEntityCfg, offset: float = 0.5):
    sensor = env.scene.sensors[sensor_cfg.name]
    return sensor.data.pos_w[:, 2].unsqueeze(1) - sensor.data.ray_hits_w[..., 2] - offset


def time_out(env):
    return env.episode_length_buf >= env.max_episode_length


def root_height_below_minimum(env, minimum_height: float, asset_cfg: SceneEntityCfg = _ROBOT):
    return env.scene[asset_cfg.name].data.root_pos_w[:, 2] < minimum_height


def image(env, sensor_cfg=None, data_type="rgb", convert_perspective_to_orthogonal=False, normalize=True):
    raise NotImplementedError("camera observations are out of scope for the fused hot path (SURVEY 8f-4)")
