#!/usr/bin/env python
"""Generate golden input/output vectors by EXECUTING THE REFERENCE'S OWN PYTHON on CPU torch tensors,
against the IsaacLab stand-in in shims/ (config carriers + trivial state accessors only):

    python tests/golden/make_golden.py <the reference's source/ directory>     # writes tests/golden/*.npz

Two kinds of fixture (DESIGN.md 5): values produced by the REFERENCE'S OWN functions (action terms, drift / elevation /
visual term functions, reset_root_state_along_track, the curriculum term, the camera post-processing), and values that pass
through an IsaacLab function restated in shims/ ([UPSTREAM-RECALL]: is_terminated_term, euler_xyz_from_quat,
quat_from_euler_xyz) -- the latter pin the oracle to the restatement, not to IsaacLab.
The vectors pin the oracle's restatement of: the action terms (ackermann_actions.py, rc_car_actions.py), the
drift reward/termination terms (mushr_drift_env_cfg.py:160-240,343-348), reset_root_state_along_track
(drifting/mdp/events.py), increase_reward_weight_over_time (curriculums.py), root_euler_xyz.  The reference is
not part of this repository, hence the committed .npz fixtures.
"""
import sys
import types
from pathlib import Path

import numpy as np
import torch

HERE = Path(__file__).resolve().parent
ROOT = HERE.parent.parent
if len(sys.argv) != 2:
    sys.exit("usage: python tests/golden/make_golden.py <the reference's source/ directory>")
REF = Path(sys.argv[1])
sys.path[:0] = [str(ROOT / "shims"), str(REF / "wheeledlab"), str(REF / "wheeledlab_assets")]
pkg = types.ModuleType("wheeledlab_tasks")          # skip wheeledlab_tasks/__init__.py (gymnasium/pxr import chain)
pkg.__path__ = [str(REF / "wheeledlab_tasks" / "wheeledlab_tasks")]
sys.modules["wheeledlab_tasks"] = pkg

import wheeledlab.envs.mdp as wmdp  # noqa: E402
from wheeledlab_tasks.common.actions import Mushr4WDActionCfg, MushrRWDActionCfg, F1Tenth4WDActionCfg  # noqa: E402
from wheeledlab_tasks.drifting import mushr_drift_env_cfg as D  # noqa: E402
from wheeledlab_tasks.drifting.mdp.events import reset_root_state_along_track  # noqa: E402
import isaaclab.utils.math as math_utils  # noqa: E402


# ---- minimal fake env ---------------------------------------------------------------------------------
class FakeData:
    pass


class FakeAsset:
    joint_names = ["back_left_wheel_throttle", "back_right_wheel_throttle", "front_left_wheel_throttle",
                   "front_right_wheel_throttle", "front_left_wheel_steer", "front_right_wheel_steer",
                   "wheel_back_left", "wheel_back_right", "wheel_front_left", "wheel_front_right", "rotator_left", "rotator_right"]

    def __init__(self):
        self.data = FakeData()
        self.captured = {}

    def find_joints(self, keys, *a, **k):
        import re
        keys = [keys] if isinstance(keys, str) else list(keys)
        ids = [i for i, n in enumerate(self.joint_names) if any(re.fullmatch(kk, n) for kk in keys)]
        return ids, [self.joint_names[i] for i in ids]

    def set_joint_velocity_target(self, target, joint_ids=None):
        self.captured["vel"] = target.clone()

    def set_joint_position_target(self, target, joint_ids=None):
        self.captured["pos"] = target.clone()

    def write_root_pose_to_sim(self, pose, env_ids=None):
        self.captured["pose"] = pose.clone()

    def write_root_velocity_to_sim(self, vel, env_ids=None):
        self.captured["velocity"] = vel.clone()


class FakeScene(dict):
    env_origins = None


class FakeRewardManager:
    def __init__(self, weights):
        self.w = dict(weights)

    def get_term_cfg(self, name):
        return types.SimpleNamespace(weight=self.w[name])

    def set_term_cfg(self, name, cfg):
        self.w[name] = cfg.weight


class FakeEnv:
    def __init__(self, n):
        self.num_envs, self.device = n, "cpu"
        self.scene = FakeScene(robot=FakeAsset())
        self.scene.env_origins = torch.zeros(n, 3)
        self.action_manager = types.SimpleNamespace(action=torch.zeros(n, 2))
        self.termination_manager = types.SimpleNamespace()
        self.max_episode_length = 250
        self.common_step_counter = 0


def golden_actions():
    g = torch.Generator().manual_seed(1)
    a = (torch.rand(512, 2, generator=g) * 4 - 2)
    a[:8] = torch.tensor([[1, 0], [0.5, 0], [-1, 0.3], [0, 1], [1, 1], [1, -1], [2, 2], [0.3, -0.7]], dtype=torch.float32)
    out = {"actions": a.numpy()}
    for name, cfgcls in (("rwd", MushrRWDActionCfg), ("fwd", Mushr4WDActionCfg), ("f1", F1Tenth4WDActionCfg)):
        cfg = cfgcls().throttle_steer
        env = FakeEnv(a.shape[0])
        term = cfg.class_type(cfg, env)
        term.process_actions(a.clone())
        term.apply_actions()
        out[name + "_processed"] = term.processed_actions.numpy().copy()
        out[name + "_wheel"] = env.scene["robot"].captured["vel"].numpy()
        out[name + "_steer"] = env.scene["robot"].captured["pos"].numpy()
        out[name + "_wheel_ids"] = np.array(term._wheel_ids)
    # the base-class true-Ackermann map (ackermann_actions.py:150-201)
    base_cfg = Mushr4WDActionCfg().throttle_steer
    env = FakeEnv(a.shape[0])
    term = wmdp.AckermannAction(base_cfg, env)
    term.process_actions(a.clone()); term.apply_actions()
    out["ack_wheel"] = env.scene["robot"].captured["vel"].numpy()
    out["ack_steer"] = env.scene["robot"].captured["pos"].numpy()
    # the other two bounding strategies of process_actions (ackermann_actions.py:126-130): 'tanh' and None (linear)
    for tag, strategy in (("tanh", "tanh"), ("none", None)):
        for name, cfgcls in (("rwd", MushrRWDActionCfg), ("fwd", Mushr4WDActionCfg)):
            cfg = cfgcls().throttle_steer
            cfg.bounding_strategy = strategy
            env = FakeEnv(a.shape[0])
            term = cfg.class_type(cfg, env)
            term.process_actions(a.clone()); term.apply_actions()
            out[f"{name}_{tag}_processed"] = term.processed_actions.numpy().copy()
            out[f"{name}_{tag}_wheel"] = env.scene["robot"].captured["vel"].numpy()
            out[f"{name}_{tag}_steer"] = env.scene["robot"].captured["pos"].numpy()
    np.savez_compressed(HERE / "actions.npz", **out)


def golden_drift_terms():
    n = 4096
    g = torch.Generator().manual_seed(2)
    pos = torch.cat([torch.rand(n, 2, generator=g) * 6 - 3, torch.zeros(n, 1)], -1)
    vel_b = torch.randn(n, 3, generator=g) * torch.tensor([2.0, 1.0, 0.2])
    ang_b = torch.randn(n, 3, generator=g) * torch.tensor([0.3, 0.3, 2.0])
    ang_w = torch.randn(n, 3, generator=g) * 2.0
    steer = torch.rand(n, 2, generator=g) * 1.2 - 0.6
    env = FakeEnv(n)
    d = env.scene["robot"].data
    d.root_pos_w, d.root_lin_vel_b, d.root_ang_vel_b, d.root_link_ang_vel_w = pos, vel_b, ang_b, ang_w
    d.joint_pos = torch.zeros(n, 12); d.joint_pos[:, 4:6] = steer
    R = D.DriftRewardsCfg()
    T = D.DriftTerminationsCfg()
    out = {"pos": pos.numpy(), "vel_b": vel_b.numpy(), "ang_b": ang_b.numpy(), "ang_w": ang_w.numpy(), "steer": steer.numpy()}
    for name in ("side_slip", "vel", "progress", "tlgr", "turn_energy", "cross_track"):
        t = getattr(R, name)
        out["f_" + name] = t.func(env, **t.params).float().numpy()
        out["w_" + name] = np.float32(t.weight)
    out["w_term_pens"] = np.float32(R.term_pens.weight)
    oob = T.out_of_bounds.func(env, **T.out_of_bounds.params)
    out["out_of_bounds"] = oob.numpy().astype(np.uint8)
    # is_terminated_term: [UPSTREAM-RECALL] -- evaluated through shims/isaaclab/envs/mdp/rewards.py (IsaacLab's function restated
    # from memory: sum of the named terms' masks times ~time_outs), NOT through the reference's own code; this fixture pins the
    # oracle to that restatement only
    env.termination_manager.active_terms = ["time_out", "out_of_bounds"]
    env.termination_manager.get_term = lambda k: oob if k == "out_of_bounds" else torch.zeros(n, dtype=torch.bool)
    env.termination_manager.time_outs = (torch.arange(n) % 7 == 0)
    out["time_outs"] = env.termination_manager.time_outs.numpy().astype(np.uint8)
    out["f_term_pens"] = R.term_pens.func(env, **R.term_pens.params).numpy()
    np.savez_compressed(HERE / "drift_terms.npz", **out)


def golden_reset_along_track():
    from isaaclab.managers import EventTermCfg
    cfg = D.DriftEventsCfg().reset_root_state
    env = FakeEnv(64)
    out = {}
    torch.manual_seed(123)
    u = torch.rand(cfg.params["num_points"])
    torch.manual_seed(123)
    term = reset_root_state_along_track(cfg, env)
    out["u"] = u.numpy()
    out["reference_poses"] = term.reference_poses.numpy()          # [20, 2, 3]: (pos xyz), (roll pitch yaw deg)
    ids = torch.arange(64)
    torch.manual_seed(77)
    idx = torch.randint(term.num_points, (64,))
    u_xy = torch.rand((64, 2)); u_yaw = torch.rand(64)
    torch.manual_seed(77)
    term(env, ids, **cfg.params)
    out["idx"], out["u_xy"], out["u_yaw"] = idx.numpy(), u_xy.numpy(), u_yaw.numpy()
    out["pose"] = env.scene["robot"].captured["pose"].numpy()
    out["velocity"] = env.scene["robot"].captured["velocity"].numpy()
    out["pos_noise"], out["yaw_noise"] = np.float32(cfg.params["pos_noise"]), np.float32(cfg.params["yaw_noise"])
    np.savez_compressed(HERE / "reset_along_track.npz", **out)


def golden_curriculum():
    C = D.DriftCurriculumCfg()
    R = D.DriftRewardsCfg()
    env = FakeEnv(4)
    env.reward_manager = FakeRewardManager({"side_slip": R.side_slip.weight, "tlgr": R.tlgr.weight, "term_pens": R.term_pens.weight})
    rows = []
    for c in range(1, 250 * 260 + 1):
        env.common_step_counter = c
        if c % 50 == 0:                      # the manager calls the terms whenever >=1 env resets; sample every 50 steps
            for name in ("more_slip", "more_tlgr", "more_term_pens"):
                t = getattr(C, name)
                t.func(env, torch.arange(4), **t.params)
            rows.append((c, env.reward_manager.w["side_slip"], env.reward_manager.w["tlgr"], env.reward_manager.w["term_pens"]))
    np.savez_compressed(HERE / "curriculum.npz", rows=np.array(rows, dtype=np.float64))


def golden_euler():
    g = torch.Generator().manual_seed(5)
    q = torch.randn(2048, 4, generator=g)
    q = q / q.norm(dim=-1, keepdim=True)
    q[:4] = torch.tensor([[1, 0, 0, 0], [0.7071068, 0, 0, 0.7071068], [0.7071068, 0, 0, -0.7071068], [0, 0, 0, 1.0]])
    env = FakeEnv(q.shape[0])
    env.scene["robot"].data.root_quat_w = q
    e = wmdp.root_euler_xyz(env)
    np.savez_compressed(HERE / "euler.npz", quat=q.numpy(), euler=e.numpy())


def golden_elevation():
    """Elevation task term functions of the reference (mushr_elevation_env_cfg.py) on random states."""
    from wheeledlab_tasks.elevation import mushr_elevation_env_cfg as E
    from isaaclab.managers import SceneEntityCfg
    n = 1024
    g = torch.Generator().manual_seed(9)
    pos = torch.cat([torch.rand(n, 2, generator=g) * 38 - 19, torch.rand(n, 1, generator=g) * 0.6 + 0.05], -1)
    rpy = torch.randn(n, 3, generator=g) * torch.tensor([0.5, 0.5, 2.0])
    # [UPSTREAM-RECALL]: quat_from_euler_xyz / euler_xyz_from_quat live in shims/isaaclab/utils/math.py (IsaacLab's functions
    # restated from memory); only root_euler_xyz itself (wheeledlab/envs/mdp/observations.py:9-12) is the reference's own code
    quat = math_utils.quat_from_euler_xyz(rpy[:, 0], rpy[:, 1], rpy[:, 2])
    vel_w = torch.randn(n, 3, generator=g) * torch.tensor([1.0, 1.0, 0.3])
    ang_w = torch.randn(n, 3, generator=g)
    cmd = torch.zeros(n, 4); cmd[:, :2] = torch.rand(n, 2, generator=g) * 8 - 4
    cmd[:64, :2] = pos[:64, :2] + (torch.rand(64, 2, generator=g) - 0.5) * 0.6          # some envs close to the goal
    omega = torch.randn(n, 4, generator=g) * 4 + 1.0
    action = torch.randn(n, 2, generator=g)
    env = FakeEnv(n)
    d = env.scene["robot"].data
    d.root_pos_w, d.root_quat_w, d.root_lin_vel_w = pos, quat, vel_w
    d.root_lin_vel_b = math_utils.quat_rotate_inverse(quat, vel_w)
    d.root_ang_vel_b = math_utils.quat_rotate_inverse(quat, ang_w)
    d.joint_vel = torch.zeros(n, 12); d.joint_vel[:, 0:4] = omega
    env.command_manager = types.SimpleNamespace(get_command=lambda name: cmd)
    env.action_manager.action = action
    out = {"pos": pos.numpy(), "quat": quat.numpy(), "vel_w": vel_w.numpy(), "ang_w": ang_w.numpy(), "cmd": cmd.numpy(),
           "omega": omega.numpy(), "action": action.numpy()}
    R, T, O = E.ElevationRewardsCfg(), E.ElevationTerminationsCfg(), E.ElevationObsCfg().policy
    out["f_goal"] = R.vel_towards_goal.func(env).numpy()
    out["f_height"] = R.height_z.func(env).numpy()
    out["f_falling"] = R.falling_penalty.func(env).float().numpy()
    out["weights"] = np.array([R.vel_towards_goal.weight, R.height_z.weight, R.falling_penalty.weight, R.termination_penalty.weight], np.float32)
    out["t_oob"] = T.cart_out_of_bounds.func(env, **T.cart_out_of_bounds.params).numpy().astype(np.uint8)
    stuck_cfg = SceneEntityCfg("robot", joint_names=".*throttle")
    # the stuck term resolves SceneEntityCfg("robot", joint_names=".*throttle") through the manager; do it by hand here
    import isaaclab.envs.mdp as imdp
    orig_joint_vel = imdp.joint_vel
    imdp.joint_vel = lambda env, asset_cfg=None: env.scene["robot"].data.joint_vel[:, 0:4]
    E.mdp.joint_vel = imdp.joint_vel
    out["t_stuck"] = T.stuck.func(env, **T.stuck.params).numpy().astype(np.uint8)
    imdp.joint_vel = orig_joint_vel; E.mdp.joint_vel = orig_joint_vel
    out["t_rollover"] = T.rollover.func(env, **T.rollover.params).numpy().astype(np.uint8)
    out["t_at_goal"] = T.at_goal.func(env, **T.at_goal.params).numpy().astype(np.uint8)
    out["o_goal"] = O.goal_relative_xyz.func(env).numpy()
    out["o_euler"] = O.world_euler_xyz.func(env).numpy()
    clip = O.base_lin_vel.clip
    out["o_linvel"] = torch.clip(O.base_lin_vel.func(env), clip[0], clip[1]).numpy()
    out["o_angvel"] = torch.clip(O.base_ang_vel.func(env), clip[0], clip[1]).numpy()
    out["o_action"] = torch.clip(O.last_action.func(env), -1, 1).numpy()
    # height map formula/sign/clip on synthetic hits: sensor.data.pos_w = ray-caster parent (base_link), hits = terrain z
    sens = types.SimpleNamespace(data=types.SimpleNamespace())
    sens.data.pos_w = pos + torch.tensor([0.0, 0.0, 0.094655])
    hits = torch.rand(n, 676, 3, generator=g) * 2.0
    hits[:, ::7, 2] = float("inf")                                        # misses
    sens.data.ray_hits_w = hits
    env.scene.sensors = {"height_scanner": sens}
    p = O.elevation_map.params
    hm = O.elevation_map.func(env, **p)
    out["hm_hits_z"] = hits[:64, :, 2].numpy(); out["hm_pos_z"] = pos[:64, 2].numpy()
    out["hm_out"] = torch.clip(hm, O.elevation_map.clip[0], O.elevation_map.clip[1])[:64].numpy()
    out["hm_offset"], out["hm_plane"] = np.float32(p["offset"]), np.float32(p["plane_init_value"])
    np.savez_compressed(HERE / "elevation_terms.npz", **out)


def golden_visual():
    """Traversability lookup (utils/traversability_utils.py) and respawn-pose formula (utils/__init__.py:188-202) of the
    Visual task, loaded by file path with stand-in modules for matplotlib / pxr (imported at module scope there)."""
    import importlib.util
    for name in ("matplotlib", "matplotlib.pyplot", "pxr"):
        sys.modules.setdefault(name, types.ModuleType(name))
    sys.modules["matplotlib"].pyplot = sys.modules["matplotlib.pyplot"]
    for k in ("Usd", "UsdGeom", "UsdPhysics", "Gf"):
        setattr(sys.modules["pxr"], k, types.SimpleNamespace())
    vdir = REF / "wheeledlab_tasks" / "wheeledlab_tasks" / "visual" / "utils"
    spec = importlib.util.spec_from_file_location("wl_visual_utils", vdir / "__init__.py", submodule_search_locations=[str(vdir)])
    vu = importlib.util.module_from_spec(spec); sys.modules["wl_visual_utils"] = vu; spec.loader.exec_module(vu)
    rng = np.random.default_rng(4)
    m = rng.random((40, 60)) < 0.3                       # [rows(y), cols(x)] non-square on purpose
    util = vu.TraversabilityHashmapUtil()
    util.set_traversability_hashmap(m.tolist(), (60, 40), (0.5, 0.5))     # map_size = (num_rows, num_cols) as the cfg passes them
    g = torch.Generator().manual_seed(3)
    pts = (torch.rand(4000, 2, generator=g) - 0.5) * torch.tensor([36.0, 26.0])
    trav = util.get_traversability(pts)
    xi, yi = util.get_map_id(pts[:, 0], pts[:, 1])
    np.random.seed(11)
    poses = vu.generate_random_poses(256, 0.5, 0.5, m.tolist(), margin=0.1)
    np.random.seed(11)
    idxs = np.random.choice(int(m.sum()), 256)
    np.savez_compressed(HERE / "visual_terms.npz", map=m, pts=pts.numpy(), trav=trav.numpy().astype(np.uint8), xi=xi.numpy(), yi=yi.numpy(),
                        poses=np.array(poses, dtype=np.float64), idxs=idxs)


def golden_camera():
    """camera_data_rgb_flattened / camera_data_rgb_flattened_aug (visual/mdp_sensors/observations.py:64-87), the reference's
    own functions run on synthetic 2-colour frames.  torchvision draws the ColorJitter / GaussianBlur parameters inside
    forward(); the two get_params hooks are pinned to known values so that the restatement can be fed the same ones."""
    import importlib.util
    import torchvision.transforms as T
    path = REF / "wheeledlab_tasks" / "wheeledlab_tasks" / "visual" / "mdp_sensors" / "observations.py"
    spec = importlib.util.spec_from_file_location("wl_visual_sensors_obs", path)
    mod = importlib.util.module_from_spec(spec); spec.loader.exec_module(mod)
    rng = np.random.default_rng(21)
    B, H, W = 6, 60, 80
    white = np.zeros((B, H, W), dtype=bool)
    for b in range(B):                                   # blobs + stripes + one all-black and one all-white-below-horizon frame
        if b == 0:
            continue
        if b == 1:
            white[b, 25:, :] = True
            continue
        for _ in range(6):
            r0, c0 = rng.integers(0, H), rng.integers(0, W)
            white[b, r0:r0 + rng.integers(2, 25), c0:c0 + rng.integers(2, 30)] = True
        white[b, :, ::7] ^= (b % 2 == 0)
    rgb = torch.from_numpy(np.repeat((white * 255).astype(np.uint8)[..., None], 3, axis=-1))
    env = types.SimpleNamespace(scene=types.SimpleNamespace(sensors={"camera": types.SimpleNamespace(data=types.SimpleNamespace(output={"rgb": rgb}))}))
    cfgp = types.SimpleNamespace(name="camera")
    raw = mod.camera_data_rgb_flattened(env, cfgp).numpy()
    augs, outs = [], []
    orders = [[0, 1, 2, 3], [1, 0, 3, 2], [3, 2, 1, 0], [2, 0, 1, 3], [1, 2, 3, 0]]
    orig_cj, orig_gb = T.ColorJitter.get_params, T.GaussianBlur.get_params
    try:
        for k, order in enumerate(orders):
            b_, c_, s_, h_ = rng.uniform(0.2, 1.8), rng.uniform(0.8, 1.2), rng.uniform(0.2, 1.8), rng.uniform(-0.5, 0.5)
            sigma = float([0.1, 0.7, 1.5, 3.3, 5.0][k])
            T.ColorJitter.get_params = staticmethod(lambda *a, _o=order, _v=(b_, c_, s_, h_): (torch.tensor(_o), *_v))
            T.GaussianBlur.get_params = staticmethod(lambda *a, _s=sigma: _s)
            out = mod.camera_data_rgb_flattened_aug(env, cfgp).numpy()
            augs.append([b_, c_, s_, h_, sigma] + order); outs.append(out)
    finally:
        T.ColorJitter.get_params, T.GaussianBlur.get_params = orig_cj, orig_gb
    np.savez_compressed(HERE / "camera_post.npz", white=white[:, H // 3:, :].reshape(B, -1).astype(np.uint8), raw=raw,
                        aug=np.array(augs, dtype=np.float32), out=np.stack(outs).astype(np.float32))


def _f32(x):
    return float(np.float32(x))


def _ulps(x):
    """x as fp32 and its two fp32 neighbours."""
    x = np.float32(x)
    return [float(x), float(np.nextafter(x, np.float32(np.inf))), float(np.nextafter(x, np.float32(-np.inf)))]


# the parameter sets of golden_device_terms: the ones the tests use plus every threshold a designed state sits on, exactly and
# one fp32 ulp either side (the state's value is exact; the threshold moves)
_Z29 = float(np.float32(np.float32(0.29) - np.float32(0.19)))          # pos.z = 0.29: z = pos.z - 0.19 in fp32
_P_UP = float(np.float32(np.pi / 2))                                   # pitch of a |sin_pitch| >= 1 quaternion (nose up)
_P_DN = float(np.float32(np.float32(-np.pi / 2) + np.float32(2 * np.pi)))   # nose down, wrapped
DEVICE_TERM_PARAMS = {
    "forward_vel": [()], "forward_wheel_spin": [()], "change_in_elevation": [()], "ascending": [()],
    "steep_penalty": [(0.3,), (0.05,)] + [(v,) for x in (0.0, _P_UP, _P_DN) for v in _ulps(x)],
    "yaw_change_onElev": [(0.5, 0.05)] + [(a, _Z29) for a in _ulps(0.5)] + [(0.25, z) for z in _ulps(_Z29)],
    "upright_penalty": [(10.0,), (40.0,)],            # + the exact angles of the designed states, added below
    "roll_on_elev": [(0.05, 0.3)] + [(_Z29, a) for a in _ulps(0.5)] + [(z, 0.25) for z in _ulps(_Z29)],
    "low_vel_penalty": [(v,) for v in _ulps(0.1)],
    "is_traversable": [()], "is_traversable_speed_scaled": [()],
    "vel_rew_trav": [(1.0, 2.0), (1.5, 2.0), (2.0, 1.0)],
    "low_speed_penalty": [(v,) for v in _ulps(0.3)] + [(v,) for v in _ulps(5.0)],
    "off_track": [(2.0, 5.0), (5.0, 15.3), (20.0, 60.0), (2.0, 4.0)],
    "roll_over": [()],
}


def golden_device_terms():
    """The 17 functions of the device-term library (csrc/wl_terms.cuh), the reference's own code from
    elevation/mushr_elevation_env_cfg.py and visual/mushr_visual_env_cfg.py, on random and designed states: every threshold
    hit exactly and one fp32 ulp either side (identity or axis-aligned quaternions there, so that both rotations are exact),
    pitch either side of 0 and |sin_pitch| >= 1, roll at pi and pi +- pi/2, r22 = +-1 with |q| != 1 and an r22 that rounds
    below -1, every off_track boundary, positions on a traversability cell edge and one ulp either side, map cells beyond
    every edge, the counter either side of bool_is_not_traversable's switch, and elevation_continuity over three-call
    sequences (its function attribute cleared before each).  euler_xyz_from_quat and matrix_from_quat come from the
    stand-in ([UPSTREAM-RECALL]); everything else is the reference's."""
    from wheeledlab_tasks.elevation import mushr_elevation_env_cfg as E
    from wheeledlab_tasks.visual import mushr_visual_env_cfg as V
    f32 = np.float32
    rng = np.random.default_rng(17)
    rows = 24                                            # square, as the reference's 500 x 500 map (get_map_id clamps x to rows)
    spacing, width = 0.5, rows * 0.5
    trav_map = rng.random((rows, rows)) < 0.45
    trav_map[0, 0], trav_map[0, 1], trav_map[-1, -1], trav_map[-1, -2] = True, False, True, False
    max_len = 50                                         # the Visual task's max_episode_length (10 s / 0.2 s)

    pos, quat, vel, ang, omega = [], [], [], [], []

    def add(p=(0.0, 0.0, 0.29), q=(1.0, 0.0, 0.0, 0.0), v=(0.0, 0.0, 0.0), w=(0.0, 0.0, 0.0), om=(0.0, 0.0, 0.0, 0.0)):
        pos.append(p); quat.append(q); vel.append(v); ang.append(w); omega.append(om)

    # random states over the map and beyond it, some on the ramp (z - 0.19 above the thresholds), random unit quaternions
    nr = 384
    rq = rng.standard_normal((nr, 4)); rq /= np.linalg.norm(rq, axis=1, keepdims=True)
    rq[: nr // 3, 1:3] *= 0.15; rq[: nr // 3] /= np.linalg.norm(rq[: nr // 3], axis=1, keepdims=True)   # mostly upright
    for i in range(nr):
        add(p=(rng.uniform(-8, 8), rng.uniform(-8, 8), rng.uniform(0.0, 0.6)), q=tuple(rq[i]), v=tuple(rng.normal(0, [1.5, 1.0, 0.5])),
            w=tuple(rng.normal(0, [1.0, 1.0, 2.0])), om=tuple(rng.normal(40, 60, 4)))
    # thresholds on identity quaternions (v_b = v_w, w_b = w_w exactly)
    for vx in _ulps(1.2) + _ulps(0.1) + _ulps(0.3) + [2.0, 3.0, 4.0] + _ulps(2.0)[1:] + _ulps(4.0)[1:]:
        add(v=(vx, 0.0, 0.0))
    add(v=(3.0, 4.0, 0.0)); add(v=(0.0, 3.0, 4.0)); add(v=(-3.0, 0.0, -4.0))
    for s in (_ulps(200.0)):
        add(om=(s, 0.0, 0.0, 0.0))
    add(om=(150.0, 25.0, 12.5, 12.5)); add(om=(-50.0, 250.0, 0.0, 0.0))
    tiny = float(np.nextafter(f32(0), f32(1)))
    for vz in (0.0, -0.0, tiny, -tiny, 1e-7, -1e-7, 0.5):
        add(v=(0.2, 0.0, vz))
    for a in _ulps(0.5) + [0.25]:
        for z in (0.29, 0.19, 0.5):
            add(p=(1.0, 1.0, z), w=(a, 0.0, a)); add(p=(1.0, 1.0, z), w=(-a, 0.0, -a))
    # Euler-angle edges: |sin_pitch| >= 1 (non-unit quaternions), pitch just either side of 0, roll at pi and pi +- pi/2
    for q in [(1.0, 0.0, 1.0, 0.0), (1.0, 0.0, -1.0, 0.0), (0.7071068, 0.0, 0.7071068, 0.0), (0.7071068, 0.0, -0.7071068, 0.0),
              (1.0, 0.0, 1e-4, 0.0), (1.0, 0.0, -1e-4, 0.0), (1.0, 0.0, 1e-8, 0.0), (1.0, 0.0, -1e-8, 0.0),
              (0.0, 1.0, 0.0, 0.0), (0.5, 0.5, 0.0, 0.0), (0.5, -0.5, 0.0, 0.0), (1.0, 1.0, 0.0, 0.0), (1.0, -1.0, 0.0, 0.0),
              (0.0, 2.0, 0.0, 0.0), (2.0, 0.0, 0.0, 0.0), (0.0, 3.0, 0.0, 0.0), (0.0, 0.0, 2.0, 0.0), (0.0, 0.6, 0.8, 0.0),
              (1e-3, 1.0, 0.0, 0.0), (1e-3, -1.0, 0.0, 0.0), (0.0, 1.0, 0.0, 1e-3), (0.0, 1.0, 0.0, -1e-3),
              (1.0, 0.5, 0.5, 0.0), (1.0, -0.5, -0.5, 0.0)]:                 # roll = +-pi/2 exactly (cos_roll = 0)
        add(q=q)              # at rest: with |q| != 1 the rotation matrix and quat_rotate_inverse scale v differently
    # r22 that rounds below -1 (arccos is NaN there): w = z = 0, x^2 + y^2 in any summation order
    found = 0
    for _ in range(20000):
        x, y = f32(rng.uniform(0.1, 3)), f32(rng.uniform(0.1, 3))
        s = f32(x * x) + f32(y * y)
        r22 = f32(1) - f32(f32(2) / s) * s
        if r22 < -1:
            add(q=(0.0, float(x), float(y), 0.0)); found += 1
            if found == 6:
                break
    # off_track boundaries: |y| = straight, |x| = corner_out_radius, the circles (3-4-5 triangles), each +- one ulp
    for (st, r) in ((2.0, 5.0), (2.0, 4.0)):
        pts = [(r, 0.0), (-r, 0.0), (r, st), (r, -st), (0.0, st), (0.0, -st), (0.0, st + r), (0.0, -st - r)]
        if r == 5.0:
            pts += [(3.0, st + 4.0), (-3.0, st + 4.0), (3.0, -st - 4.0), (4.0, st + 3.0), (-4.0, -st - 3.0)]
        for x, y in pts:
            for xx in _ulps(x):
                for yy in _ulps(y):
                    add(p=(xx, yy, 0.1))
    # |y| = straight with |x| = fp32(corner_out_radius): the straight test and the circle (r^2 rounded from double) disagree
    for x, y in ((15.3, 0.0), (-15.3, 4.9), (15.3, 5.0), (-15.3, -5.0), (0.0, 20.3), (60.0, 0.0), (0.0, -80.0), (59.9, 19.9)):
        for xx in _ulps(x):
            add(p=(xx, y, 0.1))
    # traversability: every cell edge (an integer quotient) and one ulp either side, along both axes; beyond every edge
    for k in range(-1, rows + 2):
        e = float(f32(k * spacing - width / 2 - spacing / 2))
        for ee in _ulps(e):
            add(p=(ee, 0.3, 0.1), v=(0.8, 0.0, 0.0)); add(p=(0.3, ee, 0.1), v=(0.8, 0.0, 0.0))
    for x, y in ((-100.0, 0.0), (100.0, 0.0), (0.0, -100.0), (0.0, 100.0), (-100.0, -100.0), (100.0, 100.0), (-100.0, 100.0), (100.0, -100.0)):
        add(p=(x, y, 0.1), v=(1.0, 0.0, 0.0))
    n = len(pos)
    P = torch.tensor(pos, dtype=torch.float32); Q = torch.tensor(quat, dtype=torch.float32)
    VW = torch.tensor(vel, dtype=torch.float32); WW = torch.tensor(ang, dtype=torch.float32)
    OM = torch.tensor(omega, dtype=torch.float32)

    env = FakeEnv(n)
    env.max_episode_length = max_len
    env.scene["terrain"] = types.SimpleNamespace()
    d = env.scene["robot"].data
    d.root_pos_w, d.root_quat_w, d.root_lin_vel_w, d.root_ang_vel_w = P, Q, VW, WW
    d.root_lin_vel_b = math_utils.quat_rotate_inverse(Q, VW)
    d.root_ang_vel_b = math_utils.quat_rotate_inverse(Q, WW)
    d.joint_vel = torch.zeros(n, 12); d.joint_vel[:, 0:4] = OM
    V.TraversabilityHashmapUtil().set_traversability_hashmap(trav_map.tolist(), (rows, rows), (spacing, spacing))

    params = dict(DEVICE_TERM_PARAMS)
    deg = torch.rad2deg(torch.arccos(torch.tensor([1.0, 0.0, -1.0])))          # the exact angles of the designed states
    params["upright_penalty"] = params["upright_penalty"] + [(v,) for x in deg.tolist() for v in _ulps(x)]
    names = {"forward_vel": E.forward_vel, "forward_wheel_spin": E.forward_wheel_spin, "change_in_elevation": E.change_in_elevation,
             "ascending": E.ascending, "steep_penalty": E.steep_penalty, "yaw_change_onElev": E.yaw_change_onElev,
             "upright_penalty": E.upright_penalty, "roll_on_elev": E.roll_on_elev, "low_vel_penalty": E.low_vel_penalty,
             "is_traversable": V.is_traversable, "is_traversable_speed_scaled": V.is_traversable_speed_scaled,
             "vel_rew_trav": V.vel_rew_trav, "low_speed_penalty": V.low_speed_penalty, "off_track": V.off_track,
             "roll_over": V.roll_over}
    out = {"pos": P.numpy(), "quat": Q.numpy(), "vel_w": VW.numpy(), "ang_w": WW.numpy(), "omega": OM.numpy(),
           "vel_b": d.root_lin_vel_b.numpy(), "ang_b": d.root_ang_vel_b.numpy(), "map": trav_map.astype(np.uint8),
           "spacing": np.float64(spacing), "max_episode_length": np.int64(max_len), "n_random": np.int64(nr)}
    for name, fn in names.items():
        sig = [k for k in __import__("inspect").signature(fn).parameters if k not in ("env", "asset_cfg")]
        vals = []
        for ps in params[name]:
            vals.append(fn(env, **dict(zip(sig, ps))).to(torch.float32).numpy())
        out["p_" + name] = np.array(params[name], dtype=np.float64).reshape(len(params[name]), -1)
        out["f_" + name] = np.stack(vals)
    # bool_is_not_traversable: common_step_counter either side of 1000 episodes
    ctrs = [1000 * max_len - 1, 1000 * max_len, 1000 * max_len + max_len - 1, 999 * max_len]
    vals = []
    for c in ctrs:
        env.common_step_counter = c
        vals.append(V.bool_is_not_traversable(env).to(torch.float32).numpy())
    out["t_bool_is_not_traversable"] = np.array(ctrs, np.int64)
    out["f_bool_is_not_traversable"] = np.stack(vals)
    # elevation_continuity: three calls per sequence on the same envs, the attribute cleared before each sequence
    zs = np.array([[0.29, 0.29, 0.29, 0.30, 0.50, 0.29, 0.10, 0.30, 0.29],
                   [0.29, 0.35, 0.25, 0.29, 0.40, 0.30, 0.50, 0.30, 0.29],
                   [0.29, 0.40, 0.20, 0.29, 0.30, 0.29, 0.05, 0.31, 0.30]], np.float32)
    thr = _ulps(_Z29) + [0.05, -1.0]
    ce = FakeEnv(zs.shape[1])
    cd = ce.scene["robot"].data
    seq = []
    for tz in thr:
        if hasattr(E.elevation_continuity, "prev_elevation"):
            del E.elevation_continuity.prev_elevation
        calls = []
        for k in range(zs.shape[0]):
            cd.root_pos_w = torch.zeros(zs.shape[1], 3); cd.root_pos_w[:, 2] = torch.from_numpy(zs[k])
            calls.append(E.elevation_continuity(ce, threshold_elev=tz).to(torch.float32).numpy())
        seq.append(np.stack(calls))
    del E.elevation_continuity.prev_elevation
    out["cont_z"], out["p_elevation_continuity"], out["f_elevation_continuity"] = zs, np.array(thr, np.float64)[:, None], np.stack(seq)
    np.savez_compressed(HERE / "device_terms.npz", **out)


if __name__ == "__main__":
    golden_device_terms()
    golden_camera()
    golden_visual()
    golden_elevation()
    golden_actions(); golden_drift_terms(); golden_reset_along_track(); golden_curriculum(); golden_euler()
    for f in sorted(HERE.glob("*.npz")):
        print(f.name, f.stat().st_size)
