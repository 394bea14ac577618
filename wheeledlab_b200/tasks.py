"""Task descriptions lowered to the POD ``wl_config`` the kernels consume.

Every number below restates a value from the reference configuration (file:line under
the reference's ``source/`` directory); nothing is imported from the reference at run time.

  gym ids            wheeledlab_tasks/wheeledlab_tasks/__init__.py:14-63
  Drift env          wheeledlab_tasks/wheeledlab_tasks/drifting/mushr_drift_env_cfg.py
  actions            wheeledlab_tasks/wheeledlab_tasks/common/actions.py
  observations       wheeledlab_tasks/wheeledlab_tasks/common/observations.py
  actuators          wheeledlab_assets/wheeledlab_assets/hound.py
  vehicle geometry   SURVEY.md Appendix A (decoded from Robots/UWRLL/mushr_nano_v2.usd)
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field

import numpy as np

from ._lib import WlConfig

WL_ABI_VERSION = 2
TASK_DRIFT, TASK_ELEVATION, TASK_VISUAL = 0, 1, 2
ACT_ACKERMANN, ACT_RWD, ACT_4WD = 0, 1, 2
BOUND_NONE, BOUND_CLIP, BOUND_TANH = 0, 1, 2
BL, BR, FL, FR = 0, 1, 2, 3

# mushr_drift_env_cfg.py:27-32
CORNER_IN_RADIUS, CORNER_OUT_RADIUS, LINE_RADIUS, STRAIGHT = 0.3, 2.0, 0.8, 0.8
SLIP_THRESHOLD, MAX_SPEED = 0.55, 3.0

GYM_IDS = {
    "Isaac-MushrDriftRL-v0": "drift",
    "Isaac-F1TenthDriftRL-v0": "f1tenth_drift",
    "Isaac-MushrElevationRL-v0": "elevation",
    "Isaac-MushrVisualRL-v0": "visual",
}


@dataclass
class CurriculumTerm:
    """increase_reward_weight_over_time params (wheeledlab/envs/mdp/curriculums.py:10-35)."""
    name: str
    reward_term_name: str
    increase: float
    episodes_per_increase: int = 1
    max_increases: float = math.inf


@dataclass
class TaskSpec:
    """Host-side description that accompanies a wl_config."""
    name: str
    cfg: WlConfig
    reward_names: list = field(default_factory=list)
    termination_names: list = field(default_factory=list)       # [(name, is_time_out)]
    curriculum: list = field(default_factory=list)
    obs_dim: int = 14
    action_dim: int = 2
    episode_length_s: float = 5.0
    joint_names: list = field(default_factory=list)
    heightfield: object = None                                  # float32 [ny, pitch] (elevation) / aux blob (visual)
    traversability: object = None                               # bool [rows, cols] (visual)
    # host-side (Python) MDP terms evaluated between the two halves of the staged step (env.add_*_term):
    python_reward_terms: list = field(default_factory=list)     # [(name, func, weight, params)]
    python_termination_terms: list = field(default_factory=list)  # [(name, func, time_out, params)]
    python_event_terms: list = field(default_factory=list)      # [(name, func, mode, params, interval_range_s or None)]
    # device terms (device_terms.py), evaluated by wl_step_terms: [(name, func, "reward" | "termination" | "time_out", weight, params)]
    device_terms: list = field(default_factory=list)
    # device event terms (device_events.py), applied by wl_step_terms: [(name, func, mode, params, interval_range_s or None)]
    device_events: list = field(default_factory=list)
    # the critic observation group (privileged.py, wl_critic_observe): [(name, library term, clip)] in row order; [] = none
    critic_terms: list = field(default_factory=list)
    # an Elevation row critic (DESIGN 6s, env.set_critic_observation's form): [(name, term, {"clip": .., "scale": ..})], the
    # policy row's six terms then critic-library terms; [] = none
    row_critic: list = field(default_factory=list)
    # a modified policy observation group (policy_obs.py, wl_policy_observe): [(name, library term, noise, clip, scale)] in row
    # order; [] = the built-in row.  obs_dim stays the built-in row's width; the policy side is sized by the table's
    policy_terms: list = field(default_factory=list)
    # noise, clip and scale on the Elevation / Visual row (row_terms.py, wl_set_row_terms): [(name, row term, noise, clip,
    # scale)], one per term of the built-in row in row order; [] = the built-in row
    row_terms: list = field(default_factory=list)
    # DR events in IsaacLab's mode="reset" (wl_set_reset_events): names of _lib.WL_RESET_EVENTS; [] = start-up DR only
    reset_events: list = field(default_factory=list)

    @property
    def step_dt(self) -> float:
        return float(self.cfg.sim_dt) * int(self.cfg.decimation)


MUSHR_JOINT_NAMES = [
    # throttle joints first in the wheel order used by the kernels, then steer, then suspension
    "back_left_wheel_throttle", "back_right_wheel_throttle", "front_left_wheel_throttle", "front_right_wheel_throttle",
    "front_left_wheel_steer", "front_right_wheel_steer",
    "back_left_wheel_suspension", "back_right_wheel_suspension", "front_left_wheel_suspension",
    "front_right_wheel_suspension",
]


def reference_poses_from_dists(dists: np.ndarray, track_radius: float, track_straight: float) -> np.ndarray:
    """reset_root_state_along_track.generate_reference_poses (drifting/mdp/events.py:33-100) for given arc
    lengths ``dists``.  Returns [n, 3] float32 rows (x, y, yaw_deg); the four cases are the two straights
    (heading 90 / 270 deg) and the two half circles of the stadium."""
    r, s = np.float32(track_radius), np.float32(track_straight)
    out = np.zeros((len(dists), 3), dtype=np.float32)
    pi = np.float32(math.pi)
    for k, d in enumerate(np.asarray(dists, dtype=np.float32)):
        if d < 2 * s:                                   # case 1: +x straight, heading 90 deg
            out[k] = (r, d - s, 90.0)
        elif d < 2 * s + pi * r:                        # case 2: top half-circle
            ang = (d - 2 * s) / r
            out[k] = (r * np.cos(ang), s + r * np.sin(ang), 90.0 + ang * 180.0 / pi)
        elif d < 4 * s + pi * r:                        # case 3: -x straight, heading 270 deg
            rem = d - 2 * s - pi * r
            out[k] = (-r, s - rem, 270.0)
        else:                                           # case 4: bottom half-circle
            ang2 = (d - 4 * s - pi * r) / r
            out[k] = (-r * np.cos(ang2), -s - r * np.sin(ang2), 270.0 + ang2 * 180.0 / pi)
    return out


def generate_reference_poses(num_points: int, track_radius: float, track_straight: float, seed: int) -> np.ndarray:
    """The reference draws ``torch.rand(num_points) * perimeter`` from the global generator (events.py:34-35);
    here the draw is ``numpy.random.default_rng(seed)`` so that every rank of a sharded run builds the same table."""
    perimeter = np.float32(2.0 * math.pi) * np.float32(track_radius) + np.float32(4.0) * np.float32(track_straight)
    dists = np.random.default_rng(seed).random(num_points, dtype=np.float32) * perimeter
    return reference_poses_from_dists(dists, track_radius, track_straight)


def material_buckets(num_buckets, static_range, dynamic_range, make_consistent, ground_mu_s, ground_mu_d, seed):
    """randomize_rigid_body_material bucket table (mushr_drift_env_cfg.py:98-109) lowered to Pacejka (D, C).

    Wheel material (mu_s, mu_d) combined with the ground by MULTIPLY (mushr_drift_env_cfg.py:45-49).  The tyre
    curve mu(sigma) = D sin(C atan(B sigma)) peaks at D = combined static friction and tends to
    D sin(C pi/2) = combined dynamic friction.
    """
    rng = np.random.default_rng(seed + 0x5EED)
    mu_s = rng.uniform(static_range[0], static_range[1], num_buckets)
    mu_d = rng.uniform(dynamic_range[0], dynamic_range[1], num_buckets)
    if make_consistent:
        mu_d = np.minimum(mu_d, mu_s)
    D = mu_s * ground_mu_s
    ratio = np.clip(mu_d * ground_mu_d / D, 0.0, 1.0)
    Cshape = (2.0 / math.pi) * (math.pi - np.arcsin(ratio))
    return D.astype(np.float32), Cshape.astype(np.float32)


def set_curriculum(cfg: WlConfig, reward_names, curriculum) -> None:
    """Lower CurriculumTerm list onto the cfg's on-device curriculum table."""
    if len(curriculum) > 4:
        raise NotImplementedError("at most 4 curriculum terms")
    cfg.curr_n = len(curriculum)
    for k, t in enumerate(curriculum):
        cfg.curr_slot[k] = list(reward_names).index(t.reward_term_name)
        cfg.curr_every[k] = int(t.episodes_per_increase)
        cfg.curr_max[k] = 2**31 - 1 if t.max_increases == math.inf else int(t.max_increases)
        cfg.curr_inc[k] = float(t.increase)


def _set(arr, values):
    for k, v in enumerate(values):
        arr[k] = v


def _mushr_vehicle(cfg: WlConfig) -> None:
    """MuSHR v2 lumped rigid body + wheel geometry (SURVEY Appendix A.1) and builder-chosen contact constants."""
    cfg.mass_nominal = 4.114
    # chassis inertia is "auto" in the USD (SURVEY hard part 3): box 0.44 x 0.24 x 0.12 m about the lumped COM
    m, a, b, c = 4.114, 0.44, 0.24, 0.12
    _set(cfg.inertia_nominal, (m / 12 * (b * b + c * c), m / 12 * (a * a + c * c), m / 12 * (a * a + b * b)))
    _set(cfg.com, (-0.0049, 0.0, 0.1017))
    cfg.hub_x_front, cfg.hub_x_rear, cfg.hub_y, cfg.hub_z = 0.1385, -0.158, 0.115, 0.0488
    cfg.wheel_radius = 0.0525
    cfg.wheel_inertia = 1.378e-4
    cfg.wheel_damping = 0.0
    cfg.wheel_mass_nominal, cfg.dr_base_mass_nominal = 0.1, 1.0   # wheel_link / base_link masses in the USD (Appendix A.1)
    # suspension+tyre vertical compliance: static deflection = wheel penetration at spawn (r - hub_z = 3.7 mm)
    cfg.susp_k = m * 9.81 / (4 * 0.0037)
    cfg.susp_c = 2 * 0.7 * math.sqrt(cfg.susp_k * m / 4)
    cfg.susp_travel = 0.01                       # prismatic limits +-0.01 m
    cfg.bump_k = 10 * cfg.susp_k
    cfg.comp_max = 0.03                          # force uses min(compression, 3 cm): bounded depenetration
    cfg.base_link_z = 0.094655                   # base_link above base_footprint (Appendix A.1)
    cfg.steer_inertia = 1.0e-4
    cfg.tire_B = 10.0
    cfg.tire_v0 = 0.5
    _stick_caps(cfg, m)
    cfg.gravity = 9.81


def _stick_caps(cfg: WlConfig, m: float) -> None:
    """Effective masses of the implicit-stick cap (the friction force may at most remove the contact point's slip within one
    sub-step; a larger cap over-corrects and the contact chatters with period 2 h).  The contact point sits h_c = COM height
    below the COM, so a lateral force also rolls the chassis and a longitudinal one pitches it and spins the wheel:
        1 / m_y = 4 (1/m + h_c^2 / I_xx)      (round 1 used m / 4: 2.7x too stiff for the MuSHR -> sustained roll chatter)
        1 / m_x = r_w^2 / I_w + 4 (1/m + h_c^2 / I_yy)"""
    hc2 = float(cfg.com[2]) ** 2
    cfg.tire_mx_rest = 4.0 / m + 4.0 * hc2 / float(cfg.inertia_nominal[1])
    cfg.tire_mx = 1.0 / (cfg.wheel_radius ** 2 / cfg.wheel_inertia + cfg.tire_mx_rest)
    cfg.tire_my = 1.0 / (4.0 / m + 4.0 * hc2 / float(cfg.inertia_nominal[0]))


def _f1tenth_vehicle(cfg: WlConfig) -> None:
    """F1Tenth (SURVEY Appendix A.3, Robots/F1TENTH/f1tenth.usd) + F1TENTH_4WD_ACTUATOR_CFG (wheeledlab_assets/f1tenth.py:9-27)."""
    m = 4.1565 + 4 * 1.8001 + 2 * 0.0915 + 0.368            # base_link + wheels (1.8 kg each!) + rotators + hokuyo
    cfg.mass_nominal = m
    a, b, c = 0.50, 0.30, 0.12
    _set(cfg.inertia_nominal, (m / 12 * (b * b + c * c), m / 12 * (a * a + c * c), m / 12 * (a * a + b * b)))
    _set(cfg.com, (-0.0100, 0.0, 0.03))
    cfg.hub_x_front, cfg.hub_x_rear, cfg.hub_y, cfg.hub_z = 0.194799, -0.170156, 0.142, 0.0205 - (-0.0343)
    cfg.wheel_radius = 0.055
    cfg.wheel_inertia = 0.5 * 1.8001 * 0.055 ** 2
    cfg.wheel_damping = 0.0
    cfg.wheel_mass_nominal, cfg.dr_base_mass_nominal = 1.8001, 4.1565
    cfg.hub_z = cfg.wheel_radius - 0.003                    # 3 mm static deflection at spawn
    cfg.susp_k = m * 9.81 / (4 * 0.003)
    cfg.susp_c = 2 * 0.7 * math.sqrt(cfg.susp_k * m / 4)
    cfg.susp_travel, cfg.bump_k, cfg.comp_max, cfg.base_link_z = 0.01, 10 * cfg.susp_k, 0.03, 0.0
    cfg.steer_inertia = 2.0e-3
    cfg.tire_B, cfg.tire_v0 = 10.0, 0.5
    _stick_caps(cfg, m)
    cfg.gravity = 9.81
    cfg.dc_saturation, cfg.dc_vel_limit = 1.0, 400.0
    _set(cfg.dc_effort, (0.25,) * 4)
    _set(cfg.dc_damping, (1100.0,) * 4)
    cfg.steer_kp, cfg.steer_kd, cfg.steer_vel_limit = 120.0, 8.0, 10.0
    cfg.steer_pos_limit = math.radians(45.0)


def _hound_actuators(cfg: WlConfig, drive: str) -> None:
    """HOUND_SUS_2WD_ACTUATOR_CFG / HOUND_SUS_ACTUATOR_CFG (wheeledlab_assets/hound.py:4-52)."""
    cfg.dc_saturation, cfg.dc_vel_limit = 1.05, 450.0
    if drive == "2wd":
        _set(cfg.dc_effort, (0.5, 0.5, 0.0, 0.0))          # hound.py:40-43, front passive :44-51
        _set(cfg.dc_damping, (1000.0, 1000.0, 0.0, 0.0))
    else:
        _set(cfg.dc_effort, (0.25, 0.25, 0.25, 0.25))      # hound.py:13-21
        _set(cfg.dc_damping, (1000.0,) * 4)
    cfg.steer_kp, cfg.steer_kd = 100.0, 10.0                # hound.py:5-12
    cfg.steer_vel_limit = 10.0
    cfg.steer_pos_limit = math.radians(75.0)                # joint limits [DECODED]


def drift_task(num_envs: int = 1024, seed: int = 42, env_id_offset: int = 0, randomize: bool = True,
               drive: str = "2wd", vehicle: str = "mushr") -> TaskSpec:
    """MushrDriftRLEnvCfg (drifting/mushr_drift_env_cfg.py:368-404); drive='4wd' gives the BASELINE 'HOUND 4WD' variant."""
    cfg = WlConfig()
    cfg.abi_version = WL_ABI_VERSION
    cfg.task = TASK_DRIFT
    cfg.num_envs, cfg.env_id_offset, cfg.seed = num_envs, env_id_offset, seed
    sim_dt, decimation = 0.005, 4                                      # :393-394
    cfg.sim_dt, cfg.decimation, cfg.substeps = sim_dt, decimation, 1
    episode_length_s = 5.0                                             # :396
    # ManagerBasedRLEnv.max_episode_length: ceil in Python doubles (NOT on the fp32 copy of dt) -> 250
    cfg.max_episode_length = math.ceil(episode_length_s / (sim_dt * decimation))
    cfg.episode_length_s = episode_length_s
    # actions: MushrRWDActionCfg (common/actions.py:5-24), scale re-set at :397
    cfg.action_kind = ACT_RWD if drive == "2wd" else ACT_4WD
    cfg.bounding, cfg.no_reverse = BOUND_CLIP, 1
    _set(cfg.act_scale, (MAX_SPEED, 0.488))
    _set(cfg.act_offset, (0.0, 0.0))
    cfg.base_length, cfg.base_width, cfg.wheel_radius_cfg = 0.325, 0.2, 0.05
    if vehicle == "f1tenth":
        _f1tenth_vehicle(cfg)
    else:
        _mushr_vehicle(cfg)
        _hound_actuators(cfg, drive)
    cfg.ground_mu_s, cfg.ground_mu_d = 1.1, 1.0                       # :45-49
    # startup DR (DriftEventsRandomCfg :95-154)
    cfg.dr_enable = 1 if randomize else 0
    if randomize:
        cfg.dr_num_buckets = 20
        D, Cs = material_buckets(20, (0.3, 0.5), (0.3, 0.5), True, cfg.ground_mu_s, cfg.ground_mu_d, seed)
    else:
        cfg.dr_num_buckets = 1
        D, Cs = material_buckets(1, (1.0, 1.0), (1.0, 1.0), True, cfg.ground_mu_s, cfg.ground_mu_d, seed)  # USD wheel mu
    _set(cfg.dr_bucket_D, D)
    _set(cfg.dr_bucket_C, Cs)
    _set(cfg.dr_kd_range, (10.0, 50.0))                                # :111-119
    cfg.dr_kd_mask = 0b0011 if drive == "2wd" else 0b1111              # ".*back.*throttle"
    _set(cfg.dr_mass_add, (0.3, 0.5))                                  # :145-154
    # observations (BlindObsCfg, corruption on at :399)
    cfg.enable_corruption = 1
    _set(cfg.noise_std, (0.1, 0.1, 0.5, 0.4))
    # interval pushes :121-143
    cfg.push_enable = 1 if randomize else 0
    _set(cfg.push_hf_interval, (0.1, 0.4))
    _set(cfg.push_hf_range, (0.1, 0.03, 0.3))
    _set(cfg.push_lf_interval, (0.8, 1.2))
    cfg.push_lf_yaw = 0.6
    # reset along track :82-93
    cfg.num_ref_poses, cfg.reset_pos_noise, cfg.reset_yaw_noise = 20, 0.5, 1.0
    _set(cfg.ref_poses, generate_reference_poses(20, LINE_RADIUS, STRAIGHT, seed).reshape(-1))
    # terminations / rewards
    cfg.trk_straight, cfg.trk_corner_in, cfg.trk_corner_out = STRAIGHT, CORNER_IN_RADIUS, CORNER_OUT_RADIUS
    cfg.ctd_track_radius, cfg.ctd_offset = LINE_RADIUS, -1.0          # :284-293
    cfg.slip_min_thresh, cfg.slip_max_thresh, cfg.slip_min_vel_x = 0.25, SLIP_THRESHOLD, 1.0   # :246-254
    cfg.vel_speed_target, cfg.vel_offset = MAX_SPEED, -MAX_SPEED ** 2  # :167, :256-263
    cfg.tlgr_ang_vel_thresh = 1.0                                      # :270-274
    cfg.energy_straight = STRAIGHT                                     # :276-280
    reward_names = ["side_slip", "vel", "progress", "tlgr", "turn_energy", "cross_track", "term_pens"]
    cfg.term_enable = 0b11                                             # time_out, out_of_bounds (:351-362)
    cfg.num_rew_terms = len(reward_names)
    _set(cfg.rew_weight, (10.0, -5.0, 40.0, 0.0, 20.0, -50.0, -5000.0))  # :243-299
    curriculum = [                                                     # :306-337
        CurriculumTerm("more_slip", "side_slip", 20.0, 20, 10),
        CurriculumTerm("more_tlgr", "tlgr", 10.0, 20, 5),
        CurriculumTerm("more_term_pens", "term_pens", -1000.0, 50, 5),
    ]
    set_curriculum(cfg, reward_names, curriculum)
    return TaskSpec(
        name="drift" if drive == "2wd" else "drift_4wd", cfg=cfg, reward_names=reward_names,
        termination_names=[("time_out", True), ("out_of_bounds", False)], curriculum=curriculum, obs_dim=14,
        action_dim=2, episode_length_s=episode_length_s, joint_names=list(MUSHR_JOINT_NAMES),
    )


def elevation_task(num_envs: int = 1024, seed: int = 42, env_id_offset: int = 0, heightfield=None, hf_origin=None,
                   hf_cell: float = 0.1, terrain: str = "reference") -> TaskSpec:
    """MushrElevationRLEnvCfg (elevation/mushr_elevation_env_cfg.py:437-469).  ``heightfield``: float32 [ny, nx]
    raster of the terrain top surface; default = the raster of the reference's own Terrains/huge_compact.usd
    (terrain="reference"), or a synthetic terrain with the same envelope (terrain="procedural")."""
    from .terrain import pad_pitch, procedural_heightfield, reference_heightfield
    cfg = WlConfig()
    cfg.abi_version = WL_ABI_VERSION
    cfg.task = TASK_ELEVATION
    cfg.num_envs, cfg.env_id_offset, cfg.seed = num_envs, env_id_offset, seed
    sim_dt, decimation = 0.01, 10                                      # :461-462
    cfg.sim_dt, cfg.decimation, cfg.substeps = sim_dt, decimation, 2   # integrator sub-step 5 ms
    episode_length_s = 20.0                                            # :465
    cfg.max_episode_length = math.ceil(episode_length_s / (sim_dt * decimation))
    cfg.episode_length_s = episode_length_s
    cfg.action_kind, cfg.bounding, cfg.no_reverse = ACT_4WD, BOUND_CLIP, 1      # Mushr4WDActionCfg, common/actions.py:27-48
    _set(cfg.act_scale, (3.0, 0.488))                                  # :463
    _set(cfg.act_offset, (0.0, 0.0))
    cfg.base_length, cfg.base_width, cfg.wheel_radius_cfg = 0.325, 0.2, 0.05
    _mushr_vehicle(cfg)
    _hound_actuators(cfg, "4wd")                                       # MUSHR_SUS_CFG -> HOUND_SUS_ACTUATOR_CFG
    cfg.ground_mu_s, cfg.ground_mu_d = 1.0, 1.0                        # :95-108 (combine = multiply)
    cfg.dr_enable, cfg.dr_num_buckets = 1, 5                           # :387-398: mu_s 2.0, mu_d 1.0, 5 identical buckets
    D, Cs = material_buckets(5, (2.0, 2.0), (1.0, 1.0), False, cfg.ground_mu_s, cfg.ground_mu_d, seed)
    _set(cfg.dr_bucket_D, D)
    _set(cfg.dr_bucket_C, Cs)
    _set(cfg.dr_kd_range, (10.0, 50.0))
    cfg.dr_kd_mask = 0                                                 # no randomize_actuator_gains event in this task
    _set(cfg.dr_mass_add, (0.2, 0.5))                                  # :400-407
    cfg.enable_corruption, cfg.push_enable = 0, 0                      # :85; no interval events
    _set(cfg.noise_std, (0.0, 0.0, 0.0, 0.0))
    cfg.num_ref_poses = 1
    # height-field
    if heightfield is None:
        heightfield, x0, y0, hf_cell = reference_heightfield() if terrain == "reference" else procedural_heightfield(seed)
    else:
        x0, y0 = hf_origin
    heightfield = np.ascontiguousarray(heightfield, dtype=np.float32)
    cfg.hf_ny, cfg.hf_nx = heightfield.shape
    padded = pad_pitch(heightfield)
    cfg.hf_pitch = padded.shape[1]
    cfg.hf_x0, cfg.hf_y0, cfg.hf_cell = x0, y0, hf_cell
    cfg.hf_outside_z = 0.0                                             # ground plane z = 0 outside the mesh (:120-128)
    cfg.scan_offset, cfg.scan_plane_init, cfg.scan_sensor_dz = 0.084, 0.19, 20.0   # :74-82,135
    cfg.scan_res, cfg.scan_half, cfg.obs_clip = 0.1, 1.25, 10.0        # :139 GridPatternCfg(size=[2.5,2.5], resolution=0.1)
    _set(cfg.cmd_pos_range, (-19.0, 19.0))                             # :425-435
    cfg.cmd_resample_s = 10.0
    _set(cfg.elev_reset_xy, (-19.0, 19.0))                             # :409-419
    cfg.elev_reset_yaw = 3.14
    _set(cfg.elev_reset_vel, (0.1, 0.2))
    cfg.elev_spawn_z = 0.25                                            # :97,147-149
    cfg.elev_min_height = 0.15                                         # :354-357
    cfg.elev_stuck_min_vel, cfg.elev_stuck_spin = 0.02, 5.0            # :358-364
    cfg.elev_rollover_cos = math.cos(math.radians(60.0))               # :366-369: rad2deg(acos(R22)) > 60
    cfg.elev_goal_dist = 0.5                                           # :371-374
    cfg.elev_fall_vel = 0.10                                           # :251
    cfg.elev_plane_z = 0.19                                            # :168
    reward_names = ["vel_towards_goal", "height_z", "falling_penalty", "termination_penalty"]   # :283-305
    cfg.term_enable = 0b11111                                          # time_out, cart_out_of_bounds, stuck, rollover, at_goal (:349-376)
    cfg.num_rew_terms = len(reward_names)
    _set(cfg.rew_weight, (200.0, 5000.0, 0.0, -200.0))
    curriculum = [                                                     # :311-333
        CurriculumTerm("more_goal", "vel_towards_goal", 5.0, 50, 5),
        CurriculumTerm("more_falling_pen", "falling_penalty", 1.0, 50, 10),
    ]
    set_curriculum(cfg, reward_names, curriculum)
    spec = TaskSpec(
        name="elevation", cfg=cfg, reward_names=reward_names,
        termination_names=[("time_out", True), ("cart_out_of_bounds", False), ("stuck", False), ("rollover", False),
                           ("at_goal", False)],
        curriculum=curriculum, obs_dim=689, action_dim=2, episode_length_s=episode_length_s,
        joint_names=list(MUSHR_JOINT_NAMES),
    )
    spec.heightfield = padded
    return spec


CAMERA_MODES = {None: 0, "off": 0, "raw": 1, "aug": 2}


def visual_task(num_envs: int = 1024, seed: int = 42, env_id_offset: int = 0, traversability=None, camera: str | None = None,
                randomize: bool = False) -> TaskSpec:
    """MushrVisualRLEnvCfg (visual/mushr_visual_env_cfg.py:412-439): flat plane, 4WD MuSHR, traversability-map reward,
    out-of-map termination, random traversable respawn.  ``camera``: None -> the policy observation is the 8
    proprioceptive floats only (physics-side task); "aug" -> the registered PolicyCfg (camera_data_rgb_flattened_aug, 3200
    floats, then the 8 proprio floats = 3208, :45-52) on the software pinhole camera (SURVEY 8f-4; rendering model
    builder-defined, RTX is not available); "raw" -> camera_data_rgb_flattened (no ColorJitter / GaussianBlur)."""
    from .terrain import pack_traversability, traversability_map
    cfg = WlConfig()
    cfg.abi_version = WL_ABI_VERSION
    cfg.task = TASK_VISUAL
    cfg.num_envs, cfg.env_id_offset, cfg.seed = num_envs, env_id_offset, seed
    sim_dt, decimation = 0.02, 10                                      # :435-436
    cfg.sim_dt, cfg.decimation, cfg.substeps = sim_dt, decimation, 4   # integrator sub-step 5 ms
    episode_length_s = 10.0                                            # :439
    cfg.max_episode_length = math.ceil(episode_length_s / (sim_dt * decimation))
    cfg.episode_length_s = episode_length_s
    cfg.action_kind, cfg.bounding, cfg.no_reverse = ACT_4WD, BOUND_CLIP, 1
    _set(cfg.act_scale, (3.0, 0.488))                                  # Mushr4WDActionCfg defaults (common/actions.py:44)
    _set(cfg.act_offset, (0.0, 0.0))
    cfg.base_length, cfg.base_width, cfg.wheel_radius_cfg = 0.325, 0.2, 0.05
    _mushr_vehicle(cfg)
    _hound_actuators(cfg, "4wd")
    cfg.ground_mu_s, cfg.ground_mu_d = 2.0, 2.0                        # :126-135 (combine = multiply)
    if randomize:                                                      # VisualEventsRandomCfg, :266-299
        cfg.dr_enable, cfg.dr_num_buckets = 1, 10
        D, Cs = material_buckets(10, (0.4, 0.6), (0.4, 0.6), False, cfg.ground_mu_s, cfg.ground_mu_d, seed)
        cfg.dr_mass_mode, cfg.dr_wheel_mass_enable = 1, 1              # operation="abs" on base_link (:280-288) and the wheel links (:290-299)
        _set(cfg.dr_mass_add, (1.0, 3.0))
        _set(cfg.dr_wheel_mass, (0.01, 0.3))
    else:                                                              # VisualEventsCfg: reset only
        cfg.dr_enable, cfg.dr_num_buckets = 0, 1
        D, Cs = material_buckets(1, (1.0, 1.0), (1.0, 1.0), True, cfg.ground_mu_s, cfg.ground_mu_d, seed)   # USD wheel material 1.0/1.0
        _set(cfg.dr_mass_add, (0.0, 0.0))
    _set(cfg.dr_bucket_D, D)
    _set(cfg.dr_bucket_C, Cs)
    _set(cfg.dr_kd_range, (10.0, 50.0))
    cfg.dr_kd_mask = 0
    cfg.enable_corruption, cfg.push_enable, cfg.num_ref_poses = 0, 0, 1
    if traversability is None:
        traversability = traversability_map(seed)
    blob, n_trav = pack_traversability(traversability)
    cfg.vis_rows, cfg.vis_cols = traversability.shape
    cfg.vis_n_trav = n_trav
    cfg.vis_row_spacing = cfg.vis_col_spacing = 0.5                    # :68-70
    cfg.vis_width, cfg.vis_height = cfg.vis_rows * 0.5, cfg.vis_cols * 0.5   # :113-114
    cfg.vis_spawn_z = 0.1
    if camera not in CAMERA_MODES:
        raise ValueError(f"camera must be one of {list(CAMERA_MODES)}")
    cfg.vis_cam = CAMERA_MODES[camera]
    # TiledCameraCfg, :230-246: 80 x 60, focal 1.93, apertures 3.896 x 2.453 (pinhole, square-ish pixels), ROS convention,
    # mounted at camera_link + (0.08, 0, 0) looking along the car's +x; camera_link in the root frame: SURVEY Appendix A
    cfg.vis_cam_w, cfg.vis_cam_h = 80, 60
    cfg.vis_cam_row0 = cfg.vis_cam_h // 3                              # images[:, H//3:], observations.py:67,78
    focal, h_ap, v_ap = 1.9299999475479126, 3.8959999084472656, 2.453000068664551
    cfg.vis_cam_fx, cfg.vis_cam_fy = focal * cfg.vis_cam_w / h_ap, focal * cfg.vis_cam_h / v_ap
    cfg.vis_cam_cx, cfg.vis_cam_cy = cfg.vis_cam_w / 2.0, cfg.vis_cam_h / 2.0
    _set(cfg.vis_cam_pos, (0.022995 + 0.08, 0.0175, 0.162178))         # camera_link (root frame, Appendix A.1) + OffsetCfg.pos, :242
    cfg.vis_cam_bg = 0.0                                               # no light / dome in the cfg: sky and base plane black
    cfg.vis_mesh_x0 = -cfg.vis_width / 2 - cfg.vis_row_spacing / 2     # np.linspace(-w/2, w/2, num_rows) - spacing/2, utils/__init__.py:26-28
    cfg.vis_mesh_y0 = -cfg.vis_height / 2 - cfg.vis_col_spacing / 2
    cfg.vis_mesh_dx = cfg.vis_width / (cfg.vis_rows - 1)               # (quirk: the mesh pitch is 500/499 of the reward's cell size)
    cfg.vis_mesh_dy = cfg.vis_height / (cfg.vis_cols - 1)
    cfg.vis_aug_brightness, cfg.vis_aug_contrast, cfg.vis_aug_saturation, cfg.vis_aug_hue = 0.8, 0.2, 0.8, 0.5   # observations.py:21
    _set(cfg.vis_aug_sigma, (0.1, 5.0))                                # GaussianBlur(5, sigma=(0.1, 5.0)), observations.py:23
    cam_floats = cfg.vis_cam_w * (cfg.vis_cam_h - cfg.vis_cam_row0) if cfg.vis_cam else 0
    reward_names = ["traversablility", "vel_rew"]                     # :376-387 (sic)
    cfg.term_enable = 0b11                                             # time_out, out_range (:404-409)
    cfg.num_rew_terms = len(reward_names)
    _set(cfg.rew_weight, (5.0, 7.0))
    spec = TaskSpec(name="visual", cfg=cfg, reward_names=reward_names,
                    termination_names=[("time_out", True), ("out_range", False)], curriculum=[], obs_dim=8 + cam_floats, action_dim=2,
                    episode_length_s=episode_length_s, joint_names=list(MUSHR_JOINT_NAMES))
    spec.heightfield = blob                                            # aux device blob (see header)
    spec.traversability = traversability
    return spec


def make_task(name_or_id: str, **kw) -> TaskSpec:
    name = GYM_IDS.get(name_or_id, name_or_id)
    if name == "drift":
        return drift_task(**kw)
    if name in ("drift_4wd", "hound_4wd"):
        return drift_task(drive="4wd", **kw)
    if name == "f1tenth_drift":
        spec = drift_task(drive="4wd", vehicle="f1tenth", **kw)
        spec.cfg.base_length, spec.cfg.base_width = 0.365, 0.284          # F1Tenth4WDActionCfg, common/actions.py:64-66
        spec.name = "f1tenth_drift"
        return spec
    if name == "elevation":
        return elevation_task(**kw)
    if name == "visual_random":
        return visual_task(randomize=True, **kw)
    if name == "visual":
        if name_or_id in GYM_IDS:                 # the registered task observes through the camera (PolicyCfg, :45-52)
            kw.setdefault("camera", "aug")
        return visual_task(**kw)
    raise NotImplementedError(f"task {name_or_id!r} is not implemented in this build")
