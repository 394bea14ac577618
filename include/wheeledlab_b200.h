/*
 * wheeledlab_b200.h -- C-ABI of the H100-native vectorised wheeled-robot step.
 *
 * This is the drop-in boundary for ONE path of UWRobotLearning/WheeledLab: the
 * object `gym.make(<id>, cfg=env_cfg)` returns (isaaclab.envs:ManagerBasedRLEnv,
 * reference source/wheeledlab_tasks/wheeledlab_tasks/__init__.py:14-63) and its
 * `step()/reset()/observation_manager.compute()` calls (call stack SURVEY.md 3.3).
 * The reference has no FFI of its own (pure Python down to omni.physx), so the
 * entry points below are the ones a Python binding (ctypes, see INTEGRATION.md)
 * needs to implement that surface:
 *
 *   wl_step      <- ManagerBasedRLEnv.step(action)           (train loop:
 *                   source/wheeledlab_rl/wheeledlab_rl/utils/modified_rsl_rl_runner.py:73)
 *   wl_reset     <- ManagerBasedRLEnv.reset() / _reset_idx   (wheeledlab_tasks/test/create_and_step_env.py:31)
 *   wl_observe   <- observation_manager.compute()            (modified_rsl_rl_runner.py:50)
 *   wl_startup   <- event_manager.apply(mode="startup")      (drifting/mushr_drift_env_cfg.py:95-154)
 *   wl_curriculum<- curriculum_manager.compute()             (wheeledlab/envs/mdp/curriculums.py:10-35)
 *   wl_synth_actions <- sample_space(single_action_space)    (create_and_step_env.py:37-39)
 *
 * Plain pointers and sizes only; every device pointer is caller-owned (the Python
 * host allocates with torch and passes data_ptr()); `stream` is a cudaStream_t
 * passed as void*. All functions return 0 on success, a negative WL_E* code on
 * failure, and wl_last_error() gives the message.  Nothing here falls back to CPU.
 */
#ifndef WHEELEDLAB_B200_H
#define WHEELEDLAB_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define WL_ABI_VERSION 2

/* tasks (gym ids, wheeledlab_tasks/__init__.py:14-63) */
#define WL_TASK_DRIFT     0  /* Isaac-MushrDriftRL-v0, Isaac-F1TenthDriftRL-v0 */
#define WL_TASK_ELEVATION 1  /* Isaac-MushrElevationRL-v0 */
#define WL_TASK_VISUAL    2  /* Isaac-MushrVisualRL-v0 (physics/reward side + the software camera term, vis_cam) */

/* action term kinds (wheeledlab/envs/mdp/actions/ *.py) */
#define WL_ACT_ACKERMANN 0   /* ackermann_actions.py:150-201 */
#define WL_ACT_RWD       1   /* rc_car_actions.py:12-29 */
#define WL_ACT_4WD       2   /* rc_car_actions.py:36-64 */

/* bounding strategy (ackermann_actions.py:119-133) */
#define WL_BOUND_NONE 0
#define WL_BOUND_CLIP 1
#define WL_BOUND_TANH 2

/* wheel order everywhere: [back_left, back_right, front_left, front_right]
 * (the 4WD action's own order, rc_car_actions.py:62) */
#define WL_BL 0
#define WL_BR 1
#define WL_FL 2
#define WL_FR 3

#define WL_MAX_REW_TERMS  8
#define WL_MAX_REF_POSES  32
#define WL_MAX_BUCKETS    32
#define WL_OBS_DIM_BLIND  14   /* wheeledlab_tasks/common/observations.py:19-56 */
#define WL_SCAN_SIDE      26   /* 26x26 grid, elevation/mushr_elevation_env_cfg.py:132-142 */
#define WL_SCAN_RAYS      676
#define WL_OBS_DIM_ELEV   689  /* 2+3+3+3+2+676, mushr_elevation_env_cfg.py:57-88 */

/* drift reward term slots (drifting/mushr_drift_env_cfg.py:243-299, declaration order) */
#define WL_DR_SIDE_SLIP   0
#define WL_DR_VEL         1
#define WL_DR_PROGRESS    2
#define WL_DR_TLGR        3
#define WL_DR_TURN_ENERGY 4
#define WL_DR_CROSS_TRACK 5
#define WL_DR_TERM_PENS   6
/* elevation reward term slots (mushr_elevation_env_cfg.py:283-305) */
#define WL_ER_GOAL_RATE   0
#define WL_ER_HEIGHT_Z    1
#define WL_ER_FALLING     2
#define WL_ER_TERM_PEN    3
/* visual reward term slots (visual/mushr_visual_env_cfg.py:376-387) */
#define WL_VR_TRAVERSABLE 0
#define WL_VR_FORWARD_VEL 1
#define WL_OBS_DIM_VISUAL 8    /* base_lin_vel(3) base_ang_vel(3) last_action(2); preceded by vis_cam_w*(vis_cam_h-vis_cam_row0)
                                * camera floats when vis_cam != 0 (PolicyCfg order, mushr_visual_env_cfg.py:45-52) */
#define WL_CAM_MAX_PIXELS 4096 /* kept pixels per env (80 x 40 = 3200 in the reference cfg) */

/* error codes */
#define WL_OK          0
#define WL_EINVAL     -1
#define WL_ECUDA      -2
#define WL_EUNSUPPORTED -3

/*
 * wl_config: plain-old-data description of one task instance.  Defined by an
 * X-macro so that wl_config_describe() can hand the exact field list to a
 * foreign-language binding (the ctypes mirror is generated from it).
 * XS(type, tag, name)  scalar;   XA(type, tag, name, n)  fixed array.
 */
#define WL_CONFIG_FIELDS(XS, XA)                                                                   \
    XS(int32_t, i32, abi_version)                                                                  \
    XS(int32_t, i32, task)                                                                         \
    XS(int32_t, i32, num_envs)        /* envs owned by this handle (one GPU) */                    \
    XS(int32_t, i32, env_id_offset)   /* global id of local env 0 (multi-GPU sharding) */          \
    XS(uint64_t, u64, seed)           /* mushr_drift_env_cfg.py:371 */                             \
    /* --- simulation (mushr_drift_env_cfg.py:393-396) --- */                                      \
    XS(float, f32, sim_dt)                                                                         \
    XS(int32_t, i32, decimation)                                                                   \
    XS(int32_t, i32, substeps)        /* integrator sub-steps per sim step (TGS-like) */           \
    XS(int32_t, i32, max_episode_length)                                                           \
    XS(float, f32, episode_length_s)  /* max_episode_length_s, divides the episode log (Appendix B) */ \
    XS(float, f32, gravity)                                                                        \
    /* --- action term (wheeledlab_tasks/common/actions.py) --- */                                 \
    XS(int32_t, i32, action_kind)                                                                  \
    XS(int32_t, i32, bounding)                                                                     \
    XS(int32_t, i32, no_reverse)                                                                   \
    XS(int32_t, i32, _pad0)                                                                        \
    XA(float, f32, act_scale, 2)                                                                   \
    XA(float, f32, act_offset, 2)                                                                  \
    XS(float, f32, base_length)                                                                    \
    XS(float, f32, base_width)                                                                     \
    XS(float, f32, wheel_radius_cfg)  /* action-map radius (0.05), NOT the collider radius (Q2) */ \
    /* --- vehicle (SURVEY Appendix A) --- */                                                      \
    XS(float, f32, mass_nominal)                                                                   \
    XA(float, f32, inertia_nominal, 3)                                                             \
    XA(float, f32, com, 3)            /* COM in root(base_footprint) frame */                      \
    XS(float, f32, hub_x_front)                                                                    \
    XS(float, f32, hub_x_rear)                                                                     \
    XS(float, f32, hub_y)                                                                          \
    XS(float, f32, hub_z)                                                                          \
    XS(float, f32, wheel_radius)      /* collider radius 0.0525 */                                 \
    XS(float, f32, wheel_inertia)                                                                  \
    XS(float, f32, wheel_damping)                                                                  \
    XS(float, f32, susp_k)                                                                         \
    XS(float, f32, susp_c)                                                                         \
    XS(float, f32, susp_travel)                                                                    \
    XS(float, f32, bump_k)                                                                         \
    XS(float, f32, comp_max)          /* compression used for the force is capped (depenetration) */ \
    XS(float, f32, base_link_z)       /* base_link above the root frame (ray-caster parent), A.1 */ \
    /* --- actuators (wheeledlab_assets/hound.py:4-52) --- */                                      \
    XS(float, f32, dc_saturation)                                                                  \
    XS(float, f32, dc_vel_limit)                                                                   \
    XA(float, f32, dc_effort, 4)      /* per wheel; 0 => passive (hound.py:44-51) */               \
    XA(float, f32, dc_damping, 4)     /* nominal kd per wheel (before DR) */                       \
    XS(float, f32, steer_kp)                                                                       \
    XS(float, f32, steer_kd)                                                                       \
    XS(float, f32, steer_inertia)                                                                  \
    XS(float, f32, steer_vel_limit)                                                                \
    XS(float, f32, steer_pos_limit)                                                                \
    /* --- tire / contact --- */                                                                   \
    XS(float, f32, tire_B)                                                                         \
    XS(float, f32, tire_v0)                                                                        \
    XS(float, f32, tire_mx)           /* effective mass for the longitudinal stick clamp */        \
    XS(float, f32, tire_my)                                                                        \
    XS(float, f32, tire_mx_rest)      /* 1/tire_mx - r_w^2/I_w (chassis part; the wheel part follows the wheel-mass DR) */ \
    XS(float, f32, ground_mu_s)       /* mushr_drift_env_cfg.py:45-49 (combine=multiply) */        \
    XS(float, f32, ground_mu_d)                                                                    \
    /* --- startup domain randomisation (mushr_drift_env_cfg.py:95-154) --- */                     \
    XS(int32_t, i32, dr_enable)                                                                    \
    XS(int32_t, i32, dr_num_buckets)                                                               \
    XA(float, f32, dr_bucket_D, WL_MAX_BUCKETS)   /* peak mu of bucket  (mu_s_wheel*mu_s_ground) */ \
    XA(float, f32, dr_bucket_C, WL_MAX_BUCKETS)   /* Pacejka shape s.t. asymptote = mu_d */        \
    XA(float, f32, dr_kd_range, 2)                                                                 \
    XS(int32_t, i32, dr_kd_mask)      /* bit i => wheel i gets randomised damping */               \
    XS(int32_t, i32, _pad1)                                                                        \
    XA(float, f32, dr_mass_add, 2)    /* base-mass range: += U (mode 0) or base_link mass := U (mode 1) */ \
    XS(int32_t, i32, dr_mass_mode)    /* randomize_rigid_body_mass operation: 0 "add" (drift :145-154, elevation :400-407), 1 "abs" on base_link (visual :280-288) */ \
    XS(int32_t, i32, dr_wheel_mass_enable) /* visual :290-299: wheel link masses := U(dr_wheel_mass), inertia rescaled by the mass ratio */ \
    XS(float, f32, dr_base_mass_nominal)   /* base_link mass in the USD (1.0), replaced in mode 1 */       \
    XS(float, f32, wheel_mass_nominal)     /* wheel link mass in the USD (0.1) */                          \
    XA(float, f32, dr_wheel_mass, 2)                                                               \
    /* --- observation noise (common/observations.py:27-45) --- */                                 \
    XS(int32_t, i32, enable_corruption)                                                            \
    XS(int32_t, i32, _pad2)                                                                        \
    XA(float, f32, noise_std, 4)      /* pos, euler, lin vel, ang vel */                           \
    /* --- interval pushes (mushr_drift_env_cfg.py:121-143) --- */                                 \
    XS(int32_t, i32, push_enable)                                                                  \
    XS(int32_t, i32, _pad3)                                                                        \
    XA(float, f32, push_hf_interval, 2)                                                            \
    XA(float, f32, push_hf_range, 3)  /* +-x, +-y, +-yaw */                                        \
    XA(float, f32, push_lf_interval, 2)                                                            \
    XS(float, f32, push_lf_yaw)                                                                    \
    /* --- reset along track (drifting/mdp/events.py:10-133) --- */                                \
    XS(int32_t, i32, num_ref_poses)                                                                \
    XS(float, f32, reset_pos_noise)                                                                \
    XS(float, f32, reset_yaw_noise)                                                                \
    XA(float, f32, ref_poses, 3 * WL_MAX_REF_POSES) /* x, y, yaw_deg */                            \
    /* --- drift terminations / rewards (mushr_drift_env_cfg.py:27-32,160-362) --- */              \
    XS(float, f32, trk_straight)                                                                   \
    XS(float, f32, trk_corner_in)                                                                  \
    XS(float, f32, trk_corner_out)                                                                 \
    XS(float, f32, ctd_track_radius)                                                               \
    XS(float, f32, ctd_offset)                                                                     \
    XS(float, f32, slip_min_thresh)                                                                \
    XS(float, f32, slip_max_thresh)                                                                \
    XS(float, f32, slip_min_vel_x)                                                                 \
    XS(float, f32, vel_speed_target)                                                               \
    XS(float, f32, vel_offset)                                                                     \
    XS(float, f32, tlgr_ang_vel_thresh)                                                            \
    XS(float, f32, energy_straight)                                                                \
    XS(int32_t, i32, term_enable)     /* bit j = termination term j is configured (play cfgs: terminations = None -> 0) */ \
    XS(int32_t, i32, num_rew_terms)                                                                \
    XA(float, f32, rew_weight, WL_MAX_REW_TERMS)  /* initial weights; live copy is on device */    \
    /* --- curriculum: increase_reward_weight_over_time terms (curriculums.py:10-35), evaluated ON DEVICE by the  \
     *     last CTA of every step (no host logic => the step is CUDA-graph replayable) --- */        \
    XS(int32_t, i32, curr_n)                                                                       \
    XS(int32_t, i32, _pad6)                                                                        \
    XA(int32_t, i32, curr_slot, 4)    /* reward slot of term k */                                  \
    XA(int32_t, i32, curr_every, 4)   /* episodes_per_increase */                                  \
    XA(int32_t, i32, curr_max, 4)     /* max_increases (INT32_MAX = inf) */                        \
    XA(float, f32, curr_inc, 4)       /* increase */                                               \
    /* --- elevation task (elevation/mushr_elevation_env_cfg.py) --- */                            \
    XS(int32_t, i32, hf_nx)           /* height-field raster size */                               \
    XS(int32_t, i32, hf_ny)                                                                        \
    XS(int32_t, i32, hf_pitch)        /* row pitch in floats (multiple of 4: TMA needs 16-B strides) */ \
    XS(int32_t, i32, _pad4)                                                                        \
    XS(float, f32, hf_x0)             /* world coord of sample (0,0) */                            \
    XS(float, f32, hf_y0)                                                                          \
    XS(float, f32, hf_cell)                                                                        \
    XS(float, f32, hf_outside_z)      /* physics ground outside the raster (ground plane z=0) */   \
    XS(float, f32, scan_offset)       /* 0.084, :78 */                                             \
    XS(float, f32, scan_plane_init)   /* 0.19,  :79 */                                             \
    XS(float, f32, scan_sensor_dz)    /* +20 m ray start, :135 */                                  \
    XS(float, f32, scan_res)          /* 0.1 */                                                    \
    XS(float, f32, scan_half)         /* 1.25 = (26-1)*res/2, GridPatternCfg size 2.5 */           \
    XS(float, f32, obs_clip)          /* 10, :61-82 */                                             \
    XA(float, f32, cmd_pos_range, 2)  /* +-19 m, :425-435 */                                       \
    XS(float, f32, cmd_resample_s)                                                                 \
    XA(float, f32, elev_reset_xy, 2)  /* +-19 m, :409-419 */                                       \
    XS(float, f32, elev_reset_yaw)    /* 3.14 */                                                   \
    XA(float, f32, elev_reset_vel, 2) /* U(0.1,0.2) on v_x and v_y */                              \
    XS(float, f32, elev_spawn_z)      /* 0.25, :97,147-149 */                                      \
    XS(float, f32, elev_min_height)   /* 0.15, :354-357 */                                         \
    XS(float, f32, elev_stuck_min_vel)                                                             \
    XS(float, f32, elev_stuck_spin)                                                                \
    XS(float, f32, elev_rollover_cos) /* cos(60 deg), :217-222 */                                  \
    XS(float, f32, elev_goal_dist)                                                                 \
    XS(float, f32, elev_fall_vel)                                                                  \
    XS(float, f32, elev_plane_z)      /* 0.19 in higher_elevation, :166-173 */                     \
    /* --- visual task, physics side (visual/mushr_visual_env_cfg.py); the camera term follows --- */ \
    XS(int32_t, i32, vis_rows)        /* traversability map [rows(y), cols(x)], :73-75 */          \
    XS(int32_t, i32, vis_cols)                                                                     \
    XS(int32_t, i32, vis_n_trav)      /* number of traversable cells (spawn candidates) */         \
    XS(int32_t, i32, _pad5)                                                                        \
    XS(float, f32, vis_row_spacing)   /* 0.5, :68-70 */                                            \
    XS(float, f32, vis_col_spacing)                                                                \
    XS(float, f32, vis_width)         /* num_rows*row_spacing = 250, :113-114 */                   \
    XS(float, f32, vis_height)                                                                     \
    XS(float, f32, vis_spawn_z)       /* 0.1, utils/__init__.py:188-202 + InitialPoseCfg */        \
    /* --- visual task, camera term (software pinhole camera over the 2-colour plane; SURVEY 8f-4) --- */ \
    XS(int32_t, i32, vis_cam)         /* 0 off, 1 camera_data_rgb_flattened, 2 ..._aug (mdp_sensors/observations.py:64-87) */ \
    XS(int32_t, i32, vis_cam_w)       /* 80, :234 */                                                \
    XS(int32_t, i32, vis_cam_h)       /* 60, :233 */                                                \
    XS(int32_t, i32, vis_cam_row0)    /* H // 3: rows [row0, H) are kept, observations.py:67,78 */  \
    XS(float, f32, vis_cam_fx)        /* focal_length * W / horizontal_aperture (pixels), :236-239 */ \
    XS(float, f32, vis_cam_fy)        /* focal_length * H / vertical_aperture */                    \
    XS(float, f32, vis_cam_cx)        /* W / 2 */                                                   \
    XS(float, f32, vis_cam_cy)        /* H / 2 */                                                   \
    XA(float, f32, vis_cam_pos, 3)    /* optical centre in the root frame: camera_link + offset (0.08,0,0), :242 */ \
    XS(float, f32, vis_cam_bg)        /* colour of what is not the plane mesh (sky, black base plane): 0 */ \
    XS(float, f32, vis_mesh_x0)       /* first mesh vertex: -width/2 - row_spacing/2, utils/__init__.py:26-28 */ \
    XS(float, f32, vis_mesh_y0)                                                                    \
    XS(float, f32, vis_mesh_dx)       /* vertex pitch: width / (num_rows - 1) (np.linspace), quirk: != row_spacing */ \
    XS(float, f32, vis_mesh_dy)                                                                    \
    XS(float, f32, vis_aug_brightness) /* ColorJitter(brightness=0.8, contrast=0.2, saturation=0.8, hue=0.5), observations.py:21 */ \
    XS(float, f32, vis_aug_contrast)                                                               \
    XS(float, f32, vis_aug_saturation)                                                             \
    XS(float, f32, vis_aug_hue)                                                                    \
    XA(float, f32, vis_aug_sigma, 2)  /* GaussianBlur(5, sigma=(0.1, 5.0)), observations.py:23 */  \
    /* --- derived constants: filled by wl_config_finalize() (wl_create calls it on its copy); fp32,   \
     *     formed once on the host so the kernels carry no per-step divisions for them --- */        \
    XS(float, f32, d_h)               /* sim_dt / substeps */                                      \
    XS(float, f32, d_inv_h)                                                                        \
    XS(float, f32, d_step_dt)         /* sim_dt * decimation */                                    \
    XS(float, f32, d_hkp)             /* h * steer_kp */                                           \
    XS(float, f32, d_sden)            /* 1 / (J + h kd + h^2 kp) */                                \
    XS(float, f32, d_inv_Iw)                                                                       \
    XS(float, f32, d_hI)              /* h / wheel_inertia */                                      \
    XS(float, f32, d_inv_hf_cell)     /* 1 / hf_cell (0 without a height-field) */                 \
    XS(float, f32, d_fxk)             /* tire_mx / h */                                            \
    XS(float, f32, d_fyk)                                                                          \
    XS(float, f32, d_inv_wheel_radius_cfg)                                                         \
    XS(float, f32, d_inv_dc_vel_limit)                                                             \
    XS(float, f32, d_inv_mass_nominal)                                                             \
    XA(float, f32, d_invI_nominal, 3)                                                            \
    XS(float, f32, d_vis_mesh_inv_dx) /* 1 / vis_mesh_dx (0 when the camera is off) */             \
    XS(float, f32, d_vis_mesh_inv_dy)

typedef struct wl_config {
#define WL_XS(type, tag, name) type name;
#define WL_XA(type, tag, name, n) type name[n];
    WL_CONFIG_FIELDS(WL_XS, WL_XA)
#undef WL_XS
#undef WL_XA
} wl_config;

/*
 * Device state layout.  One caller-owned buffer of wl_state_bytes() bytes holds
 * WL_NUM_GROUPS "groups"; group g is an array float4[num_envs] at byte offset
 * g * num_envs * 16, so env i reads/writes one aligned 128-bit word per group
 * and a warp touches 512 contiguous bytes (coalesced).  Component meaning:
 */
#define WL_G_POS     0  /* root_pos_w x,y,z ; episode_length_buf (int32 bits)          */
#define WL_G_QUAT    1  /* root_quat_w  w,x,y,z                                       */
#define WL_G_LINVEL  2  /* root_lin_vel_w x,y,z ; push_hf time_left                   */
#define WL_G_ANGVEL  3  /* root_ang_vel_w x,y,z ; push_lf time_left                   */
#define WL_G_WHEEL   4  /* wheel spin rate [bl,br,fl,fr] (joint_vel of *_throttle)    */
#define WL_G_STEER   5  /* steer pos L,R ; steer vel L,R                              */
#define WL_G_ACTION  6  /* action_manager.action (2) ; prev_action (2)                */
#define WL_G_SUM0    7  /* reward episode sums, terms 0-3                             */
#define WL_G_SUM1    8  /* reward episode sums, terms 4-7                             */
#define WL_G_PMASS   9  /* total mass, 1/mass, spare, spare              (DR param)   */
#define WL_G_PMU_D  10  /* Pacejka peak D per wheel                      (DR param)   */
#define WL_G_PMU_C  11  /* Pacejka shape C per wheel                     (DR param)   */
#define WL_G_PKD    12  /* DC-motor damping per wheel                    (DR param)   */
#define WL_G_CMD    13  /* elevation: goal x,y (world), heading_w, command time_left  */
#define WL_G_CMDB   14  /* elevation: command in the yaw frame x,y, heading_b, spare  */
#define WL_G_PIW    15  /* 1 / wheel spin inertia per wheel (DR param; read only when dr_wheel_mass_enable) */
#define WL_NUM_GROUPS 16

/* small global (not per-env) device block appended after the groups.  There is NO grid-wide synchronisation in a step:
 * the kernel of step t reads what step t-1 left (weights slot (t-1) & 1, accumulator row (t-1) % 3), finished envs
 * accumulate into row t % 3, and one warp (the "janitor", under the shadow of the state loads) publishes the weights of
 * step t into slot t & 1, turns row (t-1) % 3 into the extras["log"] row of step t-1 at the pointer that step
 * registered, and clears row (t+1) % 3 for the next launch.  Steps must therefore be issued with consecutive counters
 * on one stream; the host side re-arms the block (wl_step does it transparently) when a counter jumps.
 * Curriculum boundaries (counter % max_episode_length == 0): with a host-supplied counter wl_step adds a 1-thread kernel
 * after the boundary step that applies the terms in place, so the host sees the new weights as soon as the step has run
 * (the reference mutates them inside _reset_idx); with the device-resident counter the next step's threads apply them. */
typedef struct wl_globals {
    float rew_weight[2][WL_MAX_REW_TERMS]; /* live reward weights: slot (t & 1) = weights step t used (the curriculum     */
                                           /* mutates them on the way from slot to slot)                               */
    float acc[3][16];                      /* row t % 3, step t: [0..7] sum over reset envs of their episode sums,       */
                                           /* [8] #reset, [9+j] #envs whose termination term j fired                    */
    float* log_ptr[3];                     /* d_log pointer registered by step t (row t % 3); written one launch later   */
    float last_log[16];                    /* the most recent log row of a step that reset >= 1 env: IsaacLab's extras["log"] */
                                           /* persists until the next _reset_idx, so steps without a reset repeat it      */
    uint32_t step_base;                    /* device-resident base of common_step_counter (CUDA-graph replay)            */
    uint32_t ticket;                       /* CTAs finished (wl_rollout only: its K-step launch ends with a last-CTA pass)  */
    uint32_t curr_applied_t;               /* counter value whose curriculum boundary the host path already applied in place  */
    uint32_t _pad[1];
} wl_globals;
#define WL_LOG_FLOATS 16                  /* d_log: [0..7] Episode_Reward means, [8] #reset, [9+j] term counts */
/* termination term order (bit j of the per-env mask; declaration order of the reference cfgs)
 *   drift     (mushr_drift_env_cfg.py:351-362):     0 time_out, 1 out_of_bounds
 *   elevation (mushr_elevation_env_cfg.py:349-376): 0 time_out, 1 cart_out_of_bounds, 2 stuck, 3 rollover, 4 at_goal
 *   visual    (mushr_visual_env_cfg.py:404-409):    0 time_out, 1 out_range */
#define WL_MAX_TERM_TERMS 7

typedef struct wl_sim wl_sim;   /* opaque handle (host memory) */

/* ---- config ---------------------------------------------------------------- */
/* "name:tag:count:offset;..." for every wl_config field, plus "sizeof:<n>". */
const char* wl_config_describe(void);
size_t wl_config_sizeof(void);
/* device-resident counter base (wl_create zeroes it): set it / add K to it (a 1-thread kernel, capturable: the last node
 * of a replayable graph of K steps) / tell the host mirror what the device holds after graph replays the library did
 * not see (pure host call; `value` = base now in device memory). */
int wl_set_step_counter(wl_sim* sim, int64_t value, void* stream);
int wl_advance_counter(wl_sim* sim, int32_t K, void* stream);
int wl_note_device_counter(wl_sim* sim, int64_t value);
/* publish the extras["log"] row of the most recent step now (otherwise the next step's launch does it); once the flush
 * has run on the stream, the library writes that step's log buffer no more, so it may be freed or reused */
int wl_log_flush(wl_sim* sim, void* stream);
/* live reward weights (what the next step will use): device pointer to WL_MAX_REW_TERMS floats inside the state buffer */
float* wl_reward_weights(wl_sim* sim);
/* optional per-env output of wl_step / wl_step_host*: one byte of termination-term bits per env (bit j = term j fired this
 * step, order below) -- what TerminationManager.get_term(name) needs; NULL (default) disables it */
int wl_set_term_bits(wl_sim* sim, uint8_t* d_term_bits);
/* Fused rollout-slab fan-out (multi-GPU, SURVEY 8e): every output row wl_step writes (observation, reward, terminated,
 * truncated) is ALSO stored at `pointer + byte_deltas[k]` for k < n_peers -- byte_deltas[k] = base of peer k's symmetric
 * (P2P-mapped, NVLink) gathered buffer minus the base of the local one -- so the learner-facing concat of the rollout is
 * complete when the step kernels are: no separate collective.  Drift-family tasks; at most WL_MAX_PEERS (8) deltas, each a
 * multiple of 16 (WL_EINVAL otherwise: full rows leave as 16-byte stores).  n_peers = 0 switches it off, the multicast
 * delta included.
 * Only wl_step carries the fan-out, and only when it runs the 8-envs-per-CTA kernel (variant 8: Drift family, N <= 33 792,
 * default or wl_set_kernel_variant 8).  While a peer or multicast delta is set, wl_step on any other variant and
 * wl_rollout, wl_act_step, wl_act_infer_step, wl_policy_act_elu, wl_step_stage_a / _b, wl_step_host and wl_step_host_zero_copy return
 * WL_EUNSUPPORTED before any device work and leave the handle as it was.  wl_observe, wl_reset and wl_policy_act write no
 * step rows and ignore it. */
int wl_set_peer_fanout(wl_sim* sim, int32_t n_peers, const int64_t* byte_deltas);
/* NVSwitch multicast form of the fan-out: `mc_byte_delta` = (multicast alias of the symmetric buffer) - (this rank's mapping of
 * it); wl_step's variant-8 kernel then sends every full, aligned output row with ONE multimem.st that the switch replicates
 * into all ranks' buffers (NVLink egress 1x instead of (world-1)x); the rows it cannot send that way (partial CTA, unaligned
 * pointers) go peer by peer through wl_set_peer_fanout's deltas.  So the peer deltas must be set first: a nonzero delta on
 * a handle without them, or one that is not a multiple of 16, is WL_EINVAL.  0 switches it off.  The calls that refuse the
 * peer fan-out refuse this one too.  torch: _SymmetricMemory.multicast_ptr. */
int wl_set_multicast_fanout(wl_sim* sim, int64_t mc_byte_delta);
/* ManagerBasedEnv.seed(): re-key the counter-based generator for all later launches (startup draws are not repeated) */
int wl_set_seed(wl_sim* sim, uint64_t seed);
/* fill the d_* derived fields from the primary ones (idempotent). */
int wl_config_finalize(wl_config* cfg);

/* ---- lifetime -------------------------------------------------------------- */
size_t wl_state_bytes(int32_t num_envs);     /* groups + globals, 256-byte padded */
size_t wl_globals_offset(int32_t num_envs);  /* byte offset of wl_globals in the state buffer */
/* d_state: zero-initialised device buffer of wl_state_bytes(cfg->num_envs) bytes.
 * d_heightfield: float[hf_ny*hf_nx] on device (row-major: index iy*hf_nx + ix, 16-byte aligned, hf_nx % 4 == 0)
 * or NULL.  For the elevation task a TMA tensor map over it is built here.
 * Visual task: the same pointer carries the traversability data instead: int32 trav_cells[vis_n_trav] (cell id =
 * row*vis_cols + col, the spawn candidates) followed, at byte offset ((4*vis_n_trav + 15) & ~15), by
 * uint8 map[vis_rows*vis_cols] (1 = traversable). */
int wl_create(const wl_config* cfg, void* d_state, size_t state_bytes, const float* d_heightfield,
              wl_sim** out);
int wl_destroy(wl_sim* sim);
const char* wl_last_error(void);
/* compiled-for architecture string, e.g. "sm_90a" */
const char* wl_build_info(void);

/* ---- hot path -------------------------------------------------------------- */
/* startup events: material buckets / actuator gains / base mass scatter + default joint state
 * + initial interval timers (mushr_drift_env_cfg.py:95-154; EventManager startup). */
int wl_startup(wl_sim* sim, void* stream);
/* reset the listed envs (d_env_ids==NULL => all).  env ids are local int64 indices, as
 * IsaacLab passes them (_reset_idx).  `step_counter` keys the counter-based RNG. */
int wl_reset(wl_sim* sim, const int64_t* d_env_ids, int32_t n_ids, int64_t step_counter, void* stream);
/* one env.step(): action[N,2] f32 -> obs[N,obs_dim] f32, rew[N] f32, terminated[N] u8,
 * truncated[N] u8.  `step_counter` = common_step_counter BEFORE this step (>= 0), or WL_DEVICE_COUNTER_PLUS(k): the
 * counter base kept in device memory plus k -- then the call carries no per-step host value and a captured CUDA graph of
 * K such calls (k = 0..K-1) followed by wl_advance_counter(K) can be replayed.  Auto-resets finished envs (reward
 * belongs to the pre-reset state, obs to the post-reset state).  The cfg's curriculum terms are applied on the device
 * (reference: inside _reset_idx). */
#define WL_DEVICE_COUNTER (-1)
#define WL_DEVICE_COUNTER_PLUS(k) (-1 - (int64_t)(k))
/* d_log: optional float[WL_LOG_FLOATS]: mean over the envs reset in this step of each reward term's episode sum
 * divided by max_episode_length_s (RewardManager.reset -> extras["log"]), then the reset / terminated / time-out
 * counts; a step in which no env reset repeats the row of the last step that did (the reference's extras["log"] is only
 * rebuilt inside _reset_idx).  No extra kernel, no host sync, no grid-wide sync: the row of step t is written by the NEXT launch on the
 * handle (the step after it, or wl_log_flush), i.e. it is valid once that launch has completed. */
int wl_step(wl_sim* sim, const float* d_action, float* d_obs, float* d_rew, uint8_t* d_terminated,
            uint8_t* d_truncated, float* d_log, int64_t step_counter, void* stream);
/* K consecutive env.step()s in ONE launch with the state held in registers (synthetic / scripted-action rollouts:
 * wheeledlab_tasks/test/create_and_step_env.py:34-41 without the per-step host round trip).  d_actions: [K,N,2] or NULL
 * (then U[-1,1]^2 is drawn in-kernel from the counter-based generator; d_actions_out, if not NULL, receives them).
 * Outputs are [K,N,...] slabs; d_log is [K, WL_LOG_FLOATS].  Bit-identical to K wl_step calls.  With curriculum terms
 * configured, [step_counter, step_counter+K) must end at or before the next episode boundary of the global counter
 * (the boundary's weight update happens between launches).  Drift / Visual without the camera term only (the Elevation
 * scan and the Visual camera are second kernels). */
int wl_rollout(wl_sim* sim, int32_t K, const float* d_actions, float* d_actions_out, float* d_obs, float* d_rew,
               uint8_t* d_terminated, uint8_t* d_truncated, float* d_log, int64_t step_counter, void* stream);
/* env.step() for a HOST-side caller, host buffers in, host buffers out, one call:
 *   H2D  h_action[N,2] (pinned)  ->  d_action
 *   wl_step(...) writing d_obs, and reward / terminated / truncated into ONE device block d_result laid out as
 *        float rew[N] | uint8 terminated[N] | uint8 truncated[N]          (wl_result_bytes(N) bytes)
 *   D2H  d_result -> h_result (pinned, same layout), then cudaStreamSynchronize(stream).
 * Observations stay on the device (the policy lives there); pass h_obs != NULL to copy them back as well. */
size_t wl_result_bytes(int32_t num_envs);
int wl_step_host(wl_sim* sim, const float* h_action, float* d_action, float* d_obs, void* d_result, float* d_log,
                 void* h_result, float* h_obs, int64_t step_counter, void* stream);
/* Same contract, zero-copy transport: h_action / h_result must be PINNED host memory (cudaHostAlloc / torch
 * pin_memory: device-addressable under unified addressing).  The step kernel reads the actions from and writes
 * reward / terminated / truncated to host memory directly over PCIe -- no staging copies, no extra launches -- then
 * the stream is synchronised.  Bytes crossing the bus per step are identical to wl_step_host. */
 /* (h_action may be any pinned [N,2] f32 block of the caller -- it is read in place.) */
int wl_step_host_zero_copy(wl_sim* sim, const float* h_action, float* d_obs, float* d_log, void* h_result,
                           int64_t step_counter, void* stream);
/* observation_manager.compute(): re-samples the noise (SURVEY 3.4). call_idx distinguishes
 * repeated calls at the same step_counter. */
int wl_observe(wl_sim* sim, float* d_obs, int64_t step_counter, int32_t call_idx, void* stream);
/* curriculum (curriculums.py:10-35) evaluated on device so that no host sync is needed:
 * for each term t in [0,n): if any env reset during the last step, rew_weight[slot[t]] += inc[t]
 * when the host-evaluated counter conditions in fire_mask bit t hold. */
int wl_curriculum(wl_sim* sim, int32_t n_terms, const int32_t* slots, const float* increases, uint32_t fire_mask,
                  void* stream);
/* synthetic actions: U[-1,1]^2 (dist=0) or clip(N(0,1),-1,1) (dist=1) keyed by
 * (seed, global env id, step_counter); writes d_action[N,2]. */
int wl_synth_actions(wl_sim* sim, float* d_action, int64_t step_counter, int32_t dist, void* stream);
/* derived joint state for the Python articulation view: suspension pos/vel [N,4]x2 */
int wl_derive_suspension(wl_sim* sim, float* d_susp_pos, float* d_susp_vel, void* stream);
/* step-kernel geometry: 0 = auto (by num_envs and task), 1 = one thread per env, 4 = four lanes (one per wheel) per env,
 * 8 = the quad plus an auxiliary warp per 8 envs that takes everything off the dependent chain (Drift family only).
 * Results are bit-identical across variants. */
int wl_set_kernel_variant(wl_sim* sim, int32_t lanes_per_env);
/* height-scan tile staging: 1 = one TMA tile per CTA (default), 2 = TMA producer/consumer pipeline over persistent CTAs,
 * 0 = plain loads (A/B comparison); identical outputs */
int wl_set_scan_tma(wl_sim* sim, int32_t use_tma);
/* observation width for the configured task */
int32_t wl_obs_dim(const wl_sim* sim);
/* number of kernel launches issued through this handle since creation */
int64_t wl_launch_count(const wl_sim* sim);
/* number of wl_step launches through this handle that ran chained: the single-GPU duo kernel started without waiting for the
 * previous grid, because the stream's previous launch of a kernel that triggers its dependents was another env set's duo
 * step with disjoint buffers (DESIGN.md 6e) */
int64_t wl_chained_step_count(const wl_sim* sim);
/* of those, the ones that ran deep: every CTA triggered the next launch at entry and waited for the previous grid only before
 * it exited, so more than two steps of different env sets could run at once (DESIGN.md 6e) */
int64_t wl_deep_step_count(const wl_sim* sim);
/* what the most recent wl_step on this handle launched (read-only; launches nothing): the kernel variant actually used (1, 4
 * or 8 after the automatic choice; 0 before the first wl_step), the handle's step-spec key, whether the Drift-family duo
 * kernel (variant 8) ran an instantiation specialised on that key (1) or its generic body (0), and the threads per CTA of the
 * launch (duo kernel: 96 with the spacer warp, 64 without).  Any output pointer may be NULL. */
int wl_step_launch_info(const wl_sim* sim, int32_t* variant, uint32_t* spec_key, int32_t* specialised, int32_t* threads_per_cta);

/* Visual task camera term alone (wl_step / wl_observe launch it themselves when cfg.vis_cam != 0): fills the first
 * vis_cam_w * (vis_cam_h - vis_cam_row0) floats of every observation row from the current state.  d_aug = NULL draws the
 * ColorJitter / GaussianBlur parameters from the generator (one draw per call, like torchvision on a batch); otherwise
 * 9 floats on the device: brightness, contrast, saturation, hue, sigma, order[4] (fn_idx of ColorJitter.get_params). */
int wl_camera(wl_sim* sim, float* d_obs, int64_t step_counter, const float* d_aug, void* stream);

/* ---- env.step() cut in two, for HOST-SIDE (Python) reward / termination terms (SURVEY 8f-3) ----------------------------
 * IsaacLab's managers call user terms between "physics + built-in terms" and "reset" (ManagerBasedRLEnv.step: reward and
 * termination managers run on the post-physics, pre-reset state).  Stage a = sections A-E of wl_step (action, integrator,
 * counters, built-in terminations and rewards): writes the built-in reward [N] and one byte of termination bits per env
 * (bit j = built-in term j, order as listed above) and leaves the pre-reset state in the state buffer.  The caller may now
 * read the state, ADD its own reward terms to d_rew and raise its own termination flags.  Stage b = sections F-I (episode
 * log, auto-reset, commands / interval pushes, observations, last-CTA epilogue) for done = any built-in bit | extras.
 * wl_step_stage_a + wl_step_stage_b with null extras == wl_step, bit for bit. */
int wl_step_stage_a(wl_sim* sim, const float* d_action, float* d_rew, uint8_t* d_term_bits, int64_t step_counter, void* stream);
int wl_step_stage_b(wl_sim* sim, const uint8_t* d_term_bits, const uint8_t* d_extra_terminated, const uint8_t* d_extra_truncated,
                    float* d_obs, uint8_t* d_terminated, uint8_t* d_truncated, float* d_log, int64_t step_counter, void* stream);

/* ---- stage b cut once more, for HOST-SIDE (Python) event terms (IsaacLab EventTermCfg, DESIGN.md 6o) ----------------------
 * ManagerBasedRLEnv.step runs the reset events inside _reset_idx, then the interval events, then the observation manager.
 * Stage b1 = sections F and H of wl_step_stage_b with its arguments and checks (episode log, curriculum, auto-reset, the
 * built-in interval pushes; the janitor, the reset-mode DR kernel and the curriculum boundary): writes d_terminated /
 * d_truncated and leaves the post-reset, post-push state in the state buffer.  The caller may now write the state (root
 * pose and velocity, episode_length_buf, ...).  Stage b2 = sections G and I (the Elevation command, the observation and its
 * noise, the height scan / the Visual camera) formed from the state buffer as it is then, at the counter b1 was given
 * (WL_EINVAL otherwise).  wl_step_stage_b1 + wl_step_stage_b2 with nothing written between them == wl_step_stage_b, bit for
 * bit. */
int wl_step_stage_b1(wl_sim* sim, const uint8_t* d_term_bits, const uint8_t* d_extra_terminated, const uint8_t* d_extra_truncated,
                     uint8_t* d_terminated, uint8_t* d_truncated, float* d_log, int64_t step_counter, void* stream);
int wl_step_stage_b2(wl_sim* sim, float* d_obs, int64_t step_counter, void* stream);
/* Interval timers of up to WL_MAX_EVENT_TERMS host-side interval event terms (EventManager, is_global_time=False).
 * wl_set_event_timers stores the terms' interval_range_s (lo_hi[2k], lo_hi[2k+1]), allocates time_left [n_terms][N] and
 * draws it: time_left = u * (hi - lo) + lo, u = U[0,1) of the key (seed, env_id_offset + i, 0, stream 14, k).  A set-up call:
 * it synchronises the device before it returns and is not capturable.  n_terms = 0 frees the table.  WL_EINVAL, leaving
 * the handle as it was: a null handle, n_terms outside 0..8, a null table with n_terms > 0, a bound that is not finite,
 * lo < 0 or lo > hi, a peer / multicast fan-out set.
 * wl_event_timers, once per staged step between b1 and b2, per term k and env i with u_x, u_y from the key
 * (seed, env_id_offset + i, step_counter, stream 13, k): time_left = u_x * (hi - lo) + lo where d_done[i] != 0 (the envs b1
 * reset: d_terminated | d_truncated); then time_left -= step_dt; d_fired[k * N + i] = time_left < 1e-6, and where it fired
 * time_left = u_y * (hi - lo) + lo.  One launch on `stream`.  WL_EINVAL before any launch: a null argument, a counter
 * outside 0..2^31-1, no table, a fan-out set. */
#define WL_MAX_EVENT_TERMS 8
int wl_set_event_timers(wl_sim* sim, int32_t n_terms, const float* lo_hi);
int wl_event_timers(wl_sim* sim, const uint8_t* d_done, uint8_t* d_fired, int64_t step_counter, void* stream);

/* ---- device terms: the reference's unregistered reward / termination functions, in CUDA (DESIGN.md 6l) -------------------
 * A device term is one function of the library below, evaluated by a kernel between stage a and stage b with exactly the
 * semantics of the same function registered as a Python term (terminations first, then rewards in registration order,
 * fp32(f) * fp32(weight * step_dt), weight 0 skipped, per-episode sums).  E = elevation/mushr_elevation_env_cfg.py,
 * V = visual/mushr_visual_env_cfg.py; params in the order listed.  Map terms (is_traversable*, vel_rew_trav,
 * bool_is_not_traversable) need the Visual task. */
#define WL_MAX_DEVICE_TERMS 8
#define WL_TERM_E_FORWARD_VEL              1   /* clamp(v_b.x, max=1.2) */
#define WL_TERM_E_FORWARD_WHEEL_SPIN       2   /* clamp(sum of the throttle joint velocities, max=200) */
#define WL_TERM_E_CHANGE_IN_ELEVATION      3   /* v_w.z where > 0, else 0 */
#define WL_TERM_E_ASCENDING                4   /* clamp(v_w.z, min=0) */
#define WL_TERM_E_STEEP_PENALTY            5   /* (thresh_pitch) clamp(pitch - thresh, min=0), pitch wrapped to [0, 2 pi) */
#define WL_TERM_E_ELEVATION_CONTINUITY     6   /* (threshold_elev) 50 |dz| on the ramp; keeps the previous z per env */
#define WL_TERM_E_YAW_CHANGE_ON_ELEV       7   /* (threshold_yaw, threshold_z) */
#define WL_TERM_E_UPRIGHT_PENALTY          8   /* (thresh_deg) */
#define WL_TERM_E_ROLL_ON_ELEV             9   /* (z_start, roll_rate_thresh) */
#define WL_TERM_E_LOW_VEL_PENALTY         10   /* (min_vel) */
#define WL_TERM_V_IS_TRAVERSABLE          11   /* map */
#define WL_TERM_V_IS_TRAVERSABLE_SPEED_SCALED 12   /* map */
#define WL_TERM_V_VEL_REW_TRAV            13   /* map (speed_target_on_trav, speed_target_on_non_trav) */
#define WL_TERM_V_LOW_SPEED_PENALTY       14   /* (low_speed_thresh) */
#define WL_TERM_V_OFF_TRACK               15   /* (straight, corner_out_radius) */
#define WL_TERM_V_BOOL_IS_NOT_TRAVERSABLE 16   /* map; 0 until common_step_counter // max_episode_length reaches 1000 */
#define WL_TERM_V_ROLL_OVER               17   /* roll - pi in (-pi/2, pi/2), roll wrapped to [0, 2 pi) */
#define WL_TERM_KINDS                     18
#define WL_TERM_ROLE_REWARD      0
#define WL_TERM_ROLE_TERMINATION 1   /* fires when the value is nonzero: terminated */
#define WL_TERM_ROLE_TIME_OUT    2   /* fires when the value is nonzero: truncated */
typedef struct wl_term_desc {
    int32_t kind;        /* WL_TERM_* */
    int32_t role;        /* WL_TERM_ROLE_* */
    double weight;       /* reward weight (ignored for terminations); Python's weight * step_dt is formed in double */
    double params[4];    /* the function's parameters as Python floats (unused ones 0) */
} wl_term_desc;
/* Store the handle's device terms (at most WL_MAX_DEVICE_TERMS, evaluated in this order) and allocate their per-env
 * state: the reward terms' episode sums (zero) and elevation_continuity's previous elevation (unset: its first call sees
 * no change).  The state survives env resets, as the reference's function attribute does; it is per handle.  n = 0 clears
 * the table.  A set-up call: it allocates, clears the state and synchronises the device before it returns, and it is not
 * capturable.  The old table's buffers are freed only after the new ones are ready (a failure leaves the handle as it
 * was), so a graph captured with the old table must be captured again.  Refused before any device work: WL_EINVAL for a
 * null handle, n outside 0..8, a null table with n > 0, an unknown kind or role, a non-finite weight or parameter;
 * WL_EUNSUPPORTED for a map term on a task other than Visual. */
int wl_set_device_terms(wl_sim* sim, const wl_term_desc* terms, int32_t n_terms);
/* One env.step with the device terms: stage a, the term kernel, stage b (and the height scan / camera).  Same arguments
 * as wl_step, plus d_term_log: NULL or float[WL_MAX_DEVICE_TERMS] on the device receiving, per term in table order,
 * Episode_Reward/<name> (the mean episode sum over the envs done in this step / max_episode_length_s) or
 * Episode_Termination/<name> (the number of done envs where it fired), then zeros; written by this call, fixed-order
 * sums.  With device event terms (wl_set_device_events) stage b runs cut: stage b1, the reset-mode DR kernel, the device
 * events, stage b2.  With neither terms nor events the call is wl_step itself and d_term_log is not written.
 * step_counter is a host counter or WL_DEVICE_COUNTER_PLUS(k), so K calls and wl_advance_counter(K) form a replayable
 * graph.  WL_EINVAL for a null argument or a misaligned action /
 * obs, WL_EUNSUPPORTED while a peer / multicast fan-out is set, before any device work. */
int wl_step_terms(wl_sim* sim, const float* d_action, float* d_obs, float* d_rew, uint8_t* d_terminated, uint8_t* d_truncated,
                  float* d_log, float* d_term_log, int64_t step_counter, void* stream);
/* Device pointer to uint8[N]: bit k = device term k fired in the most recent wl_step_terms (NULL without terms). */
uint8_t* wl_device_term_masks(const wl_sim* sim);

/* ---- device event terms: IsaacLab's push_by_setting_velocity in CUDA (DESIGN.md 6p) --------------------------------------
 * Per term k, for the envs it fires for, each world-frame root velocity component c (0..5: x, y, z, roll, pitch, yaw) gains
 * u * (hi_c - lo_c) + lo_c (fp32, no fma), u = U[0,1) of the key (seed, env_id_offset + i, step, stream 15, k) for c = 0..3
 * (.x .. .w) and (seed, env_id_offset + i, step, stream 15, 8 + k) for c = 4, 5 (.x, .y); terms apply in table order.  A
 * reset-mode term fires for the envs the step reset (terminated | truncated); an interval-mode term for the envs whose
 * timer ran out, the timer of wl_event_timers (redraw at reset, count down by step_dt, fire below 1e-6, redraw) on a slot
 * of its own: the j-th interval term of the table uses timer index j in the keys of streams 13 and 14.  Every task
 * integrates all six components (chassis_integrate: 3-D velocity and body rates on the plane and on the height-field), so
 * no component needs a zero range. */
#define WL_MAX_DEVICE_EVENTS 8
#define WL_EVENT_MODE_RESET    1
#define WL_EVENT_MODE_INTERVAL 2
typedef struct wl_device_event_desc {
    int32_t mode;                 /* WL_EVENT_MODE_* */
    float interval_range_s[2];    /* (lo, hi) of an interval term: finite, 0 <= lo <= hi; ignored in reset mode */
    float velocity_range[6][2];   /* (lo, hi) per component x, y, z, roll, pitch, yaw: finite, lo <= hi */
} wl_device_event_desc;
/* Store the handle's device event terms and draw the interval terms' timers (key (seed, env_id_offset + i, 0, stream 14,
 * j)).  n = 0 clears the table.  A set-up call: it allocates, draws and synchronises the device before it returns, and it
 * is not capturable; a failure leaves the handle as it was.  Refused before any device work: WL_EINVAL for a null handle,
 * n outside 0..8, a null table with n > 0, an unknown mode, a bound that is not finite, lo > hi, a negative interval bound,
 * a peer / multicast fan-out set.  With a table, wl_step_terms applies the terms each step (stage a, the device terms,
 * stage b1, the reset-mode DR kernel, wl_device_events, stage b2), and wl_step, wl_act_step, wl_act_infer_step, wl_rollout
 * and the staged step refuse the handle (WL_EUNSUPPORTED): they would step it without the events. */
int wl_set_device_events(wl_sim* sim, const wl_device_event_desc* table, int32_t n_terms);
/* The device event terms of one step on the handle's state, after stage b1 wrote d_terminated / d_truncated: one launch
 * on `stream`, capturable.  step_counter: the counter b1 was given (host value 0..2^31-1 or WL_DEVICE_COUNTER_PLUS(k)).
 * WL_EINVAL before any launch: a null argument, a counter out of range, no table, a fan-out set. */
int wl_device_events(wl_sim* sim, const uint8_t* d_terminated, const uint8_t* d_truncated, int64_t step_counter, void* stream);

/* ---- the step before env.step(): the policy (SURVEY 8f-1) ---------------------------------------------------------
 * alg.act(obs) of the rollout loop (modified_rsl_rl_runner.py:72; rsl_rl ActorCritic with the reference's sizes,
 * drifting/config/agents/mushr/rsl_rl_ppo_cfg.py:12-17: actor and critic 64x64 ELU MLPs, Gaussian head with a learned
 * std) FUSED in front of the env step: one launch = value + action mean + sampled action + log-prob + the whole step.
 * Weights are a caller-owned device blob of fp32 in INPUT-MAJOR (transposed) layout, per net:
 *     W1t[ceil4(obs_dim)][64] b1[64]  W2t[64][64] b2[64]  W3t[64][out] b3[out]   (actor: out = 2, critic: out = 1;
 *     rows obs_dim.. of W1t are zero padding)
 * blob = actor net | critic net | std[2]; every block starts 16-byte aligned (wl_policy_blob_floats gives offsets).
 * a = mean + std * z, z ~ N(0,1) from the counter-based generator (stream 9, keyed by global env id and step). */
typedef struct wl_policy_out {
    float* actions;      /* [N,2] sampled actions (also what the env step consumes) */
    float* mean;         /* [N,2] */
    float* log_prob;     /* [N]   sum over action dims */
    float* value;        /* [N]   */
} wl_policy_out;
/* offsets (in floats) of the 13 arrays inside the blob for observation width obs_dim; returns the total float count */
int32_t wl_policy_blob_floats(int32_t obs_dim, int32_t offsets[13]);
int wl_act_step(wl_sim* sim, const float* d_obs_in, const float* d_policy_blob, wl_policy_out out, float* d_obs,
                float* d_rew, uint8_t* d_terminated, uint8_t* d_truncated, float* d_log, int64_t step_counter, void* stream);
/* wl_act_step for playback (rsl_rl ActorCritic.act_inference, the runner's get_inference_policy()): the action is the
 * actor mean -- no critic, no policy noise, no log-prob -- then the same env step, PDL trigger / wait, janitor and episode
 * log as wl_act_step.  Writes d_actions [N,2] (8-byte aligned) and nothing else of a wl_policy_out; equals
 * wl_actor_mean(d_obs_in, ..., WL_ACTIVATION_ELU) bit for bit, which equals the mean wl_act_step stores.  The tasks of
 * wl_act_step only (obs_dim <= 16, not Elevation). */
int wl_act_infer_step(wl_sim* sim, const float* d_obs_in, const float* d_policy_blob, float* d_actions, float* d_obs,
                      float* d_rew, uint8_t* d_terminated, uint8_t* d_truncated, float* d_log, int64_t step_counter, void* stream);
/* wl_act_step's policy without the env step, for a step launched separately (e.g. the staged step, whose Python terms run
 * between wl_step_stage_a and wl_step_stage_b): for every env of `sim`, the actor mean, critic value, sampled action and
 * log-prob of d_obs_in [N, obs_dim] under the ELU network in d_policy_blob into `out`.  For the same d_obs_in, blob, seed,
 * env_id_offset and step_counter (a host counter or WL_DEVICE_COUNTER_PLUS(k)) all four outputs equal what wl_act_step
 * stores, bit for bit.  One launch; no env state, janitor or episode log is touched, and it does not trigger dependents
 * early, so a step launched after it with PDL waits for every action.  Returns before any launch: WL_EINVAL for a null
 * or misaligned pointer (blob 16 bytes, actions / mean 8, obs_in / log_prob / value 4) or a counter out of range;
 * WL_EUNSUPPORTED for obs_dim > 16 or while a peer / multicast fan-out is set (the step after it refuses it too). */
int wl_policy_act_elu(wl_sim* sim, const float* d_obs_in, const float* d_policy_blob, wl_policy_out out, int64_t step_counter,
                      void* stream);

/* ---- the asymmetric actor-critic: a privileged critic observation group (DESIGN.md 6m) -----------------------------------
 * rsl_rl's ActorCritic(num_actor_obs, num_critic_obs, ...) fed from extras["observations"]["critic"]
 * (modified_rsl_rl_runner.py:51, :77-82): the actor reads the policy row, the critic a second row of its own width.
 * Drift family only (policy obs_dim <= 16, ELU), critic width Dc <= WL_MAX_CRITIC_OBS.
 *
 * The critic row is the concatenation, in table order, of terms of this library; no noise is ever added:
 *   kind                         width  content
 *   WL_CRITIC_ROOT_POS_W           3    root position, world frame          } the BlindObsCfg terms, formed as the
 *   WL_CRITIC_ROOT_EULER_XYZ       3    roll, pitch, yaw wrapped to [0, 2pi) } policy row forms them, without the
 *   WL_CRITIC_BASE_LIN_VEL         3    linear velocity, body frame          } noise draw
 *   WL_CRITIC_BASE_ANG_VEL         3    angular velocity, body frame         }
 *   WL_CRITIC_LAST_ACTION          2    action_manager.action                }
 *   WL_CRITIC_JOINT_VEL            4    throttle joint velocities [bl, br, fl, fr] (state group WL_G_WHEEL)
 *   WL_CRITIC_JOINT_POS            2    steer joint positions L, R (WL_G_STEER)
 *   WL_CRITIC_WHEEL_FRICTION       4    per-wheel peak friction coefficient of the env's DR bucket (WL_G_PMU_D)
 *   WL_CRITIC_BASE_MASS            1    total mass (WL_G_PMASS)
 *   WL_CRITIC_MOTOR_DAMPING        4    DC-motor damping per wheel (WL_G_PKD)
 * clip > 0 clamps the term's floats to [-clip, clip] (ObservationTermCfg.clip, symmetric); 0 = no clip. */
#define WL_MAX_CRITIC_OBS   32
#define WL_MAX_CRITIC_TERMS 16
#define WL_CRITIC_ROOT_POS_W      1
#define WL_CRITIC_ROOT_EULER_XYZ  2
#define WL_CRITIC_BASE_LIN_VEL    3
#define WL_CRITIC_BASE_ANG_VEL    4
#define WL_CRITIC_LAST_ACTION     5
#define WL_CRITIC_JOINT_VEL       6
#define WL_CRITIC_JOINT_POS       7
#define WL_CRITIC_WHEEL_FRICTION  8
#define WL_CRITIC_BASE_MASS       9
#define WL_CRITIC_MOTOR_DAMPING  10
#define WL_CRITIC_KINDS          11
typedef struct wl_critic_term {
    int32_t kind;        /* WL_CRITIC_* */
    float clip;          /* symmetric clip bound, 0 = none */
} wl_critic_term;
/* Store the handle's critic table (a host-side set-up call: nothing is launched or allocated, and a failure leaves the
 * handle as it was).  n_terms = 0 clears it.  WL_EINVAL: null handle, n_terms outside 0..WL_MAX_CRITIC_TERMS, a null table
 * with n_terms > 0, an unknown kind, a negative or non-finite clip, a total width above WL_MAX_CRITIC_OBS;
 * WL_EUNSUPPORTED: a task other than the Drift family.  A graph captured with the old table keeps the old table. */
int wl_set_critic_terms(wl_sim* sim, const wl_critic_term* terms, int32_t n_terms);
/* Dc: the width of the critic row (0 with no table; a row critic's 689 + extra width) */
int32_t wl_critic_obs_dim(const wl_sim* sim);

/* ---- reset-mode domain randomisation (IsaacLab EventTermCfg mode="reset", DESIGN.md 6n) --------------------------------
 * The start-up events of wl_startup draw each env's parameters once.  A bit set here redraws that event's parameters for
 * every env a call resets: the envs a step auto-reset (wl_step, wl_step_host, wl_step_host_zero_copy, wl_act_step,
 * wl_act_infer_step, wl_step_stage_b, wl_step_terms) and the env_ids of wl_reset (all envs when NULL).  The draw is
 * wl_startup's with the key (seed, env_id_offset + i, t, stream 12, k) instead of (.., 0, stream 6, k), t being the step
 * counter of the call that reset the env (decoded from the device counter for WL_DEVICE_COUNTER_PLUS), k = 0 buckets,
 * 1 gains, 2 base mass, 3 wheel masses.  The total mass is formed as wl_startup forms it, from the nominal mass: a
 * component whose bit is clear is recomputed from its start-up key, so it keeps its start-up value bit for bit.
 *   WL_RESET_EV_MATERIAL        randomize_rigid_body_material: WL_G_PMU_D, WL_G_PMU_C  (needs dr_enable)
 *   WL_RESET_EV_ACTUATOR_GAINS  randomize_actuator_gains: WL_G_PKD                   (needs dr_enable, dr_kd_mask != 0)
 *   WL_RESET_EV_BASE_MASS       randomize_rigid_body_mass on the base: WL_G_PMASS     (needs dr_enable)
 *   WL_RESET_EV_WHEEL_MASS      randomize_rigid_body_mass on the wheels: WL_G_PMASS, WL_G_PIW (needs dr_wheel_mass_enable)
 * A host-side set-up call kept per handle: nothing is launched.  With mask 0 (the default) no call launches anything new.
 * With a non-zero mask every call listed above launches one more kernel on its stream after its own work, and wl_rollout
 * returns WL_EUNSUPPORTED.  WL_EINVAL, leaving the handle as it was: a null handle, an unknown bit, a bit whose event the
 * config does not have.  A graph captured with the old mask keeps the old mask. */
#define WL_RESET_EV_MATERIAL       1u
#define WL_RESET_EV_ACTUATOR_GAINS 2u
#define WL_RESET_EV_BASE_MASS      4u
#define WL_RESET_EV_WHEEL_MASS     8u
int wl_set_reset_events(wl_sim* sim, uint32_t mask);
/* the handle's mask (0 for a null handle) */
uint32_t wl_reset_events(const wl_sim* sim);
/* d_critic_obs [N, Dc] (rows leave as 16-byte stores when it is 16-byte aligned) from the state the most recent step / reset left -- after wl_step, the
 * post-reset state its observation row was formed from.  One launch, no generator and no counter; capturable.  For a handle
 * whose noise_std are all 0 the five BlindObsCfg columns equal the policy row of wl_step (as fp32 values; a -0 that the
 * policy row's "+ 0 * z" turned into +0 stays -0 here).  WL_EINVAL: a null pointer or one not 4-byte aligned, no table. */
int wl_critic_observe(wl_sim* sim, float* d_critic_obs, void* stream);
/* wl_policy_blob_floats with the critic's W1t block sized by critic_obs_dim: W1t[ceil4(critic_obs_dim)][64].  For
 * critic_obs_dim == obs_dim the offsets and the total are wl_policy_blob_floats's. */
int32_t wl_policy_blob_floats_asym(int32_t obs_dim, int32_t critic_obs_dim, int32_t offsets[13]);
/* wl_policy_act_elu with the critic's first layer fed from d_critic_obs_in [N, critic_obs_dim] and a blob laid out by
 * wl_policy_blob_floats_asym(obs_dim, critic_obs_dim).  The same CTA geometry, blob copies, layer tiles, head butterfly and
 * policy noise: actions, mean and log-prob equal wl_policy_act_elu's for the same d_obs_in and actor blocks bit for bit,
 * whatever the critic input is, and with critic_obs_dim == obs_dim and d_critic_obs_in == d_obs_in the value does too.
 * Returns before any launch as wl_policy_act_elu does, plus WL_EINVAL for a null / misaligned d_critic_obs_in or
 * critic_obs_dim outside 1..WL_MAX_CRITIC_OBS. */
int wl_policy_act_asym(wl_sim* sim, const float* d_obs_in, const float* d_critic_obs_in, int32_t critic_obs_dim,
                       const float* d_policy_blob, wl_policy_out out, int64_t step_counter, void* stream);

/* ---- a modified policy observation group for the Drift family (DESIGN.md 6q) ----------------------------------------------
 * IsaacLab's ObservationManager.compute for the "policy" group of a cfg whose terms differ from BlindObsCfg's: the row is
 * the concatenation, in table order, of terms of the critic library (WL_CRITIC_*, with the widths listed there) and
 *   WL_POLICY_PROJECTED_GRAVITY    3    the gravity direction (0, 0, -1) in the body frame (projected_gravity_b)
 * Per term, in this order: the value; additive noise, only when the config's enable_corruption is set -- Gaussian
 * (x + mean) + std * z, or uniform (x + u * (n_max - n_min)) + n_min, u in [0, 1); the clip [lo, hi] (r_clamp); the scale
 * (x * s), one value or one per float.  Each step is one fp32 operation, no fma.  Parameters are the cfg's Python floats;
 * each is rounded to fp32 as torch rounds a scalar operand, n_max - n_min is formed in double first, as Python forms it.
 * Noise keys of column j (0-based in the row), env global id g, step counter t:
 *   Gaussian, j < 12:  Philox (seed, g, t, 0, j / 4) after a step and (seed, g, t, 7, 3 call_idx + j / 4) for an observe
 *                      call: the built-in row's own keys, so BlindObsCfg's five terms through a table are the built-in row;
 *                      lanes (x, y) -> Box-Muller -> columns 4b, 4b + 1, lanes (z, w) -> 4b + 2, 4b + 3
 *   otherwise:         Philox (seed, g, t, 16, 16 (call_idx + 1) + 8 u + j / 4), u = 1 for uniform noise, call_idx = -1
 *                      after a step; word j % 4 (U[0,1) from its top 24 bits) or its Box-Muller lane as above
 * so no two columns, steps or call indices share a key. */
#define WL_MAX_POLICY_OBS   32
#define WL_MAX_POLICY_TERMS 16
#define WL_POLICY_PROJECTED_GRAVITY 11
#define WL_POLICY_OBS_KINDS 12
#define WL_NOISE_NONE     0
#define WL_NOISE_GAUSSIAN 1   /* noise_params = (mean, std) */
#define WL_NOISE_UNIFORM  2   /* noise_params = (n_min, n_max) */
#define WL_POLICY_OBS_AFTER_STEP (-1)   /* wl_policy_observe's call_idx for the row of the step just taken */
typedef struct wl_policy_term {
    int32_t kind;             /* WL_CRITIC_* or WL_POLICY_PROJECTED_GRAVITY */
    int32_t noise;            /* WL_NOISE_* */
    double noise_params[2];
    int32_t clip;             /* 1: clamp to [clip_range[0], clip_range[1]] */
    int32_t n_scale;          /* 0: no scale; 1: scale[0] for every float; the term's width: scale[k] for float k */
    double clip_range[2];
    double scale[4];
} wl_policy_term;
/* Store the handle's policy table (a host-side set-up call: nothing is launched or allocated; every term is checked before
 * the table is replaced, so a failure leaves the handle as it was).  n_terms = 0 clears it.  WL_EINVAL: a null handle,
 * n_terms outside 0..WL_MAX_POLICY_TERMS, a null table with n_terms > 0, an unknown kind or noise model, n_scale not 0, 1 or
 * the width, a parameter that is not finite, a total width above WL_MAX_POLICY_OBS; WL_EUNSUPPORTED: a task other than the
 * Drift family, a peer / multicast fan-out set.  With a table, wl_act_step, wl_act_infer_step and wl_rollout return
 * WL_EUNSUPPORTED (they hand their next call the built-in row); wl_step, wl_step_terms and wl_observe still write the
 * built-in row.  wl_policy_act_elu, wl_policy_act and wl_policy_act_asym read rows of width Dp (and a blob laid out for
 * Dp) from then on: the policy is trained and played on the table's row.  A graph captured with the old table keeps the old
 * table. */
int wl_set_policy_terms(wl_sim* sim, const wl_policy_term* terms, int32_t n_terms);
/* Dp: the width of the policy row (0 with no table) */
int32_t wl_policy_obs_dim(const wl_sim* sim);
/* d_out [N, Dp] (16-byte stores when it is 16-byte aligned) from the state the most recent step / reset left -- after a
 * step, the post-reset state of the envs it reset.  call_idx = WL_POLICY_OBS_AFTER_STEP: the row of the step taken at
 * step_counter; call_idx >= 0: the row of wl_observe(step_counter, call_idx).  step_counter: a host value 0..2^31-1 or
 * WL_DEVICE_COUNTER_PLUS(k).  One launch, capturable.  Before any launch: WL_EINVAL for a null pointer or one not 4-byte
 * aligned, no table, a counter out of range, call_idx outside -1..2^27-1; WL_EUNSUPPORTED while a peer / multicast
 * fan-out is set (only the built-in row carries it). */
int wl_policy_observe(wl_sim* sim, int64_t step_counter, int32_t call_idx, float* d_out, void* stream);

/* ---- noise, clip and scale on the Elevation and Visual policy rows (DESIGN.md 6r) ----------------------------------------
 * The row terms of a handle: one wl_policy_term per term of the task's built-in policy row, in row order, with the term's
 * kind at that position --
 *   Elevation (689 floats):  WL_ROW_GOAL_RELATIVE_XYZ (2), WL_CRITIC_ROOT_EULER_XYZ (3), WL_CRITIC_BASE_LIN_VEL (3),
 *                            WL_CRITIC_BASE_ANG_VEL (3), WL_CRITIC_LAST_ACTION (2), WL_ROW_WORLD_HEIGHT_MAP (676)
 *   Visual (camera floats, then 8): WL_CRITIC_BASE_LIN_VEL (3), WL_CRITIC_BASE_ANG_VEL (3), WL_CRITIC_LAST_ACTION (2)
 * With row terms every entry that writes the row forms those columns from the raw values (goal_relative_xyz with its
 * nan_to_num, the euler angles, the body-frame velocities, the unclipped last action; a ray that misses is +inf), then per
 * term, as ObservationManager.compute does and with wl_policy_term's arithmetic and rounding (6q): additive noise only when
 * the config's enable_corruption is set, the clip, the scale.  The camera floats are not touched.  So the registered
 * group is the row terms {none, none, clip +-obs_clip, clip +-obs_clip, clip +-1, clip +-obs_clip}, and the Visual tail
 * {none, none, clip +-1}.
 * Noise keys of row column j (0-based: 0..688 on Elevation, 0..7 in the Visual tail), env global id g, step counter t
 * (decoded from WL_DEVICE_COUNTER_PLUS(k)):
 *   Philox (seed, g, t, 17, 512 (call_idx + 1) + 256 u + j / 4), u = 1 for uniform noise, call_idx = -1 for the row a
 *   step writes and wl_observe's call_idx (0..2^23-2) for an observe call; word j % 4 gives U[0,1) from its top 24 bits,
 *   lanes (x, y) -> Box-Muller -> columns 4b, 4b + 1 and lanes (z, w) -> 4b + 2, 4b + 3 give N(0, 1)
 * so no two columns, noise kinds, steps or call indices share a key, and the draws do not depend on launch geometry. */
#define WL_ROW_GOAL_RELATIVE_XYZ 12
#define WL_ROW_WORLD_HEIGHT_MAP  13
#define WL_ROW_TERMS_ELEVATION   6
#define WL_ROW_TERMS_VISUAL      3
/* Store the handle's row terms (a host-side set-up call: nothing is launched; every term is checked before anything is
 * replaced, so a failure leaves the handle as it was).  n_terms = 0 clears them; otherwise it is the task's term count.
 * WL_EINVAL: a null handle, a null table with n_terms > 0, n_terms neither 0 nor the count, a kind other than the row's term
 * at that position, an unknown noise model, n_scale not 0, 1 or the width (the map: 0 or 1), a parameter that is not
 * finite.  WL_EUNSUPPORTED: the Drift family (wl_set_policy_terms), a peer / multicast fan-out set, scan mode 2.
 * With row terms wl_step, wl_step_terms, wl_step_stage_b / _b2, wl_observe, wl_step_host and wl_step_host_zero_copy write
 * the modified row; wl_act_step, wl_act_infer_step and wl_rollout return WL_EUNSUPPORTED, and so does wl_set_scan_tma(2).
 * wl_observe takes call_idx 0..2^23-2 (WL_EINVAL otherwise).  A graph captured with the old terms keeps the old terms. */
int wl_set_row_terms(wl_sim* sim, const wl_policy_term* terms, int32_t n_terms);
/* the number of row terms (0: none) */
int32_t wl_row_terms(const wl_sim* sim);
/* The row critic of an Elevation handle (DESIGN.md 6s): a critic row of Dc = 689 + (extra width) floats -- the Elevation
 * row's six terms in row order (row_terms, as for wl_set_row_terms), noise-free, each with its own clip and scale, then
 * the critic-library terms `extra` (WL_CRITIC_*, as wl_set_critic_terms, at most WL_MAX_CRITIC_OBS floats), so Dc is in
 * 689..721.  wl_critic_obs_dim gives Dc and wl_critic_observe writes [N, Dc]: the ray-cast again, from the state the most
 * recent step / reset left, with no draw; a ray that misses is +inf before the map term's clip, as in the policy row.  The
 * policy row (built-in or row terms, noisy or not) is not touched.  A host-side set-up call: everything is checked before
 * anything is replaced.  n_row_terms = 0 (and n_extra = 0) clears it.  WL_EINVAL: a null handle, a null table with a count
 * above 0, wl_set_row_terms's refusals, a term with noise, a height-map term without a clip, extra columns without the row
 * terms, more than WL_MAX_CRITIC_TERMS extra terms, an unknown extra kind, a negative or non-finite extra clip, extra columns
 * wider than WL_MAX_CRITIC_OBS.  WL_EUNSUPPORTED: a task other than Elevation.  A handle without a row critic behaves as
 * before; one with both a row critic and a wl_set_critic_terms table cannot exist (that call refuses Elevation). */
int wl_set_row_critic(wl_sim* sim, const wl_policy_term* row_terms, int32_t n_row_terms, const wl_critic_term* extra, int32_t n_extra);

/* ---- the step after the rollout: returns / advantages over the [T, N] slab (SURVEY 8f-2) ---------------------------
 * rsl_rl RolloutStorage.compute_returns as called at modified_rsl_rl_runner.py:116 [UPSTREAM-RECALL], with the time-out
 * bootstrap of PPO.process_env_step (rewards += gamma * values * time_outs) folded in when d_time_outs != NULL:
 *   delta_t = r_t + (1 - done_t) * gamma * V_{t+1} - V_t ;  A_t = delta_t + (1 - done_t) * gamma * lam * A_{t+1}
 *   returns_t = A_t + V_t ; advantages_t = A_t          (V_T = d_last_values; no normalisation here)
 * All arrays are [T, N] row-major (env fastest), exactly the rollout-slab layout; one thread per env walks t = T-1..0. */
int wl_gae(const float* d_rewards, const float* d_values, const float* d_last_values, const uint8_t* d_dones,
           const uint8_t* d_time_outs, float gamma, float lam, float* d_returns, float* d_advantages, int32_t T,
           int32_t N, void* stream);

/* ---- the runner's episode statistics over the [T, N] slab ------------------------------------------------------------
 * rsl_rl's runner bookkeeping (modified_rsl_rl_runner.py:55-63, :99-109): per env, for t = 0..T-1,
 *   cur_return += rewards[t] (fp32, in t order); cur_length += 1;
 *   if terminated[t] | truncated[t]: append (cur_return, cur_length) to a deque(maxlen=100), envs in ascending id order
 *   (the nonzero() order); then cur_return = cur_length = 0.
 * d_cur_return / d_cur_length [N] f32 carry the running episodes between calls; *d_stats carries the deque (zero-fill it
 * for an empty one) and receives the outputs.  The means are fp64 sums over the ring, oldest episode first, divided by
 * `fill` (statistics.mean of the deque; 0 while it is empty).  Two launches, no float atomics, no host sync, graph-
 * capturable; results are bit-identical run to run.  T in 1..4096. */
#define WL_EPISODE_RING 100
typedef struct wl_episode_stats_state {
    float ring_return[WL_EPISODE_RING];  /* finished episodes: slot (head - fill + k) mod 100 holds the k-th oldest */
    float ring_length[WL_EPISODE_RING];
    int32_t fill;                        /* episodes in the ring (<= 100) */
    int32_t head;                        /* slot the next finished episode goes to */
    int32_t finished;                    /* output: episodes that finished during the last call */
    int32_t _pad;
    double mean_return;                  /* output: mean of ring_return over the ring (Train/mean_reward) */
    double mean_length;                  /* output: mean of ring_length (Train/mean_episode_length) */
} wl_episode_stats_state;
/* workspace for wl_episode_stats (a (return, length) cell per (t, env) and a done word per (t, 32 envs)); 0 on bad T / N */
size_t wl_episode_stats_workspace_bytes(int32_t T, int32_t N);
int wl_episode_stats(const float* d_rewards, const uint8_t* d_terminated, const uint8_t* d_truncated, int32_t T, int32_t N,
                     float* d_cur_return, float* d_cur_length, wl_episode_stats_state* d_stats, void* d_workspace,
                     size_t workspace_bytes, void* stream);

/* ---- the learner's data-parallel step for the small policy networks (SURVEY 8f-2) --------------------------------------
 * Gradient all-reduce fused with the Adam update, one kernel over peer memory: d_grads[r] = rank r's flat fp32 gradient
 * (this rank's own buffer and the P2P-mapped buffers of its peers, e.g. slices of one torch symmetric-memory allocation; the
 * same rank order on every rank, so every replica forms the identical mean); d_param / d_m / d_v = this rank's flat
 * parameters and Adam moments, n floats each.  `step` = 1, 2, ... (bias correction).  The caller brackets the launch with
 * barriers (all gradients written before; none overwritten until every rank has read them).  n_ranks = 1 is plain Adam.
 * The betas are doubles so that 1 - beta^step and 1 - beta are formed from the caller's values as torch.optim.Adam forms
 * them (an fp32 0.999 puts 1 - 0.999^step ~1.3e-5 off); they reach the update as fp32, as torch's kernels receive them. */
int wl_dp_adam_step(float* d_param, float* d_m, float* d_v, int32_t n_ranks, const float* const* d_grads, float lr, double beta1,
                    double beta2, float eps, float weight_decay, int32_t step, int32_t n, void* stream);

/* ---- the learner: rsl_rl PPO.update() for the Drift-family actor-critic, trained in the act-step blob in place -------
 * rsl_rl PPO.update() (modified_rsl_rl_runner.py:118; rsl-rl-lib >= 2.3.0) [UPSTREAM-RECALL] on the network wl_act_step
 * runs (obs_dim <= 16, [64, 64] ELU actor and critic, 2 actions, learned per-action std), with the weights, gradients
 * and Adam moments all in the blob layout above.  One call enqueues the whole update (epochs x mini-batches), never
 * syncs the host and is graph-capturable:
 *   advantages normalised once over the batch ((A - mean) / (unbiased std + 1e-8), computed on the fly; the caller's
 *   tensor is not modified); old sigma = the blob's std when the update starts; per mini-batch i (rows
 *   perm[i*B .. (i+1)*B), B = batch / num_mini_batches, the same permutation every epoch): clipped surrogate +
 *   value_loss_coef * (clipped) value loss - entropy_coef * entropy, gradient (torch autograd semantics at max / clamp
 *   edges), KL-adaptive learning rate, clip_grad_norm_(max_grad_norm), Adam (0.9, 0.999, 1e-8).
 * The reduction order depends only on (batch, the device's SM count): results are bit-identical run to run. */
typedef struct wl_ppo_params {
    int32_t obs_dim;
    int32_t batch;                  /* T * N rows of the slab */
    int32_t num_learning_epochs;
    int32_t num_mini_batches;
    float clip_param;
    float value_loss_coef;
    float entropy_coef;
    float max_grad_norm;
    float desired_kl;
    int32_t adaptive;               /* 1: schedule "adaptive" (the KL rule moves the device lr); 0: "fixed" */
    int32_t use_clipped_value_loss;
    int32_t _pad;
} wl_ppo_params;
typedef struct wl_ppo_batch {      /* device arrays over the [T*N] rows, slab order (row = t*N + n) */
    const float* obs;               /* [batch, obs_dim] the observations the actions were drawn from */
    const float* actions;           /* [batch, 2] */
    const float* values;            /* [batch] values at collection time (the value-clip anchor) */
    const float* log_prob;          /* [batch] log-probabilities at collection time */
    const float* mean;              /* [batch, 2] action means at collection time */
    const float* returns;           /* [batch] */
    const float* advantages;        /* [batch] un-normalised */
    const int64_t* perm;            /* [batch] a permutation of 0..batch-1 (torch.randperm) */
} wl_ppo_batch;
/* the device state d_state[wl_ppo_state_floats()] (fp32; the caller zero-fills it and sets [0] = initial learning rate):
 *   [0] learning rate  [1] Adam step count  [2..3] old std  [4] advantage mean  [5] advantage std
 *   [6] sum of surrogate losses  [7] sum of value losses  [8] sum of entropies (over this update's mini-batches)
 *   [9] the last mini-batch's KL  [10..] per mini-batch (KL, learning rate used) pairs of the last update, up to
 *   WL_PPO_MAX_UPDATES mini-batches */
#define WL_PPO_MAX_UPDATES 256
int32_t wl_ppo_state_floats(void);
/* workspace for wl_ppo_update on the current device (it holds one gradient row per CTA; 0 and wl_last_error() on error) */
size_t wl_ppo_workspace_bytes(int32_t obs_dim, int32_t batch, int32_t num_mini_batches);
/* d_blob / d_adam_m / d_adam_v: wl_policy_blob_floats(obs_dim) floats each, 16-byte aligned; the moments start zero.
 * Padding rows and columns of the blob stay exactly zero.  The workspace's first blob-sized row holds the last
 * mini-batch's reduced gradient (before clipping) after the call. */
int wl_ppo_update(const wl_ppo_params* params, const wl_ppo_batch* batch, float* d_blob, float* d_adam_m, float* d_adam_v,
                  float* d_state, void* d_workspace, size_t workspace_bytes, void* stream);

/* wl_ppo_update for the asymmetric network (rsl_rl PPO.update() with privileged observations): the critic's layer-1 forward
 * and its dW1 are taken over d_critic_obs [batch, critic_obs_dim] (slab order, gathered through the same perm), the blob /
 * moments are laid out by wl_policy_blob_floats_asym(params->obs_dim, critic_obs_dim).  The same three kernels per
 * mini-batch, no float atomics, rows summed in CTA order; padding floats of the blob are never stepped.  With
 * critic_obs_dim == obs_dim and d_critic_obs == batch->obs it leaves blob, moments and state equal to wl_ppo_update's, bit
 * for bit.  critic_obs_dim in 1..WL_MAX_CRITIC_OBS; d_critic_obs 4-byte aligned; otherwise wl_ppo_update's checks. */
size_t wl_ppo_asym_workspace_bytes(int32_t obs_dim, int32_t critic_obs_dim, int32_t batch, int32_t num_mini_batches);
int wl_ppo_update_asym(const wl_ppo_params* params, const wl_ppo_batch* batch, const float* d_critic_obs, int32_t critic_obs_dim,
                       float* d_blob, float* d_adam_m, float* d_adam_v, float* d_state, void* d_workspace, size_t workspace_bytes,
                       void* stream);

/* ---- the wide actor-critic: the Elevation / Visual policy and its PPO update -------------------------------------------
 * The same network and blob layout as above with ReLU instead of ELU between the layers (the reference's Elevation and
 * Visual agent cfgs, activation="relu"), for any obs_dim in 1..4096.  FP32 FFMA throughout; layer 1 runs as a K-chunked
 * SGEMM, since W1t no longer fits in shared memory.
 * wl_policy_act: for every env of `sim`, the actor mean, critic value, sampled action and log-prob of d_obs_in [N, obs_dim]
 * into `out`.  The noise is wl_act_step's (seed, env_id_offset + env, decoded step_counter -- device-relative counters
 * included), so a = mean + std * z matches it bit for bit for the same mean.  One launch; it does not step the env:
 * follow it with wl_step(out.actions, ..., the same step_counter). */
int wl_policy_act(wl_sim* sim, const float* d_obs_in, const float* d_policy_blob, wl_policy_out out, int64_t step_counter,
                  void* stream);
/* The actor mean alone, for any batch and without a sim handle: d_mean [n,2] (8-byte aligned) = actor(d_obs [n, obs_dim])
 * under the network in d_policy_blob (16-byte aligned).  activation WL_ACTIVATION_ELU: wl_act_step's network, obs_dim
 * 1..16, bit for bit the mean wl_act_step stores for the same rows; WL_ACTIVATION_RELU: obs_dim 1..4096, bit for bit the
 * mean wl_policy_act stores.  One launch on the device that holds d_mean; it does not trigger dependents early, so a
 * wl_step after it waits for every mean.  Bad arguments (n < 1, obs_dim out of range, ELU with obs_dim > 16, an unknown
 * activation, a null or misaligned pointer) return WL_EINVAL / WL_EUNSUPPORTED before any device call. */
#define WL_ACTIVATION_ELU 0
#define WL_ACTIVATION_RELU 1
int wl_actor_mean(const float* d_obs, int32_t n, int32_t obs_dim, const float* d_policy_blob, int32_t activation, float* d_mean,
                  void* stream);
/* rsl_rl PPO.update() on that network: the semantics, structs and d_state layout of wl_ppo_update (relu'(z) = (h > 0), 0
 * at z == 0 as torch's threshold_backward).  Per mini-batch: the gathered layer-1 forward, layers 2-3 and the loss with
 * back-propagation to layer 1's pre-activation, the gathered split-K dW1, then wl_ppo_update's reduce and Adam step.
 * No float atomics: results are bit-identical run to run for a given (batch, SM count).  The workspace also holds the
 * mini-batch's layer-1 activations and their gradients (2 x batch / num_mini_batches x 128 floats). */
size_t wl_ppo_wide_workspace_bytes(int32_t obs_dim, int32_t batch, int32_t num_mini_batches);
int wl_ppo_update_wide(const wl_ppo_params* params, const wl_ppo_batch* batch, float* d_blob, float* d_adam_m, float* d_adam_v,
                       float* d_state, void* d_workspace, size_t workspace_bytes, void* stream);

/* ---- behaviour cloning: rsl_rl's Distillation.update() on the student actor (DESIGN.md 6t) -------------------------------
 * The student is the actor of a blob laid out by wl_policy_blob_floats(obs_dim) (its critic blocks unused), trained to the
 * teacher's actions: d_obs [T, N, obs_dim] and d_teacher_actions [T, N, 2] (slab order, row = t*N + n).  The loss of step
 * t is mse(actor(obs_t), teacher_actions_t), the mean over N x 2 elements.  The epochs walk the T steps in order, counting
 * across epochs; after every gradient_length-th step the summed loss of those steps is back-propagated through the actor,
 * clip_grad_norm_(max_grad_norm) is applied when max_grad_norm > 0, and Adam (0.9, 0.999, 1e-8, the fixed learning rate
 * d_state[0]) steps the actor's parameters.  Steps after the last full chunk are evaluated but not stepped.  The critic
 * blocks, the std and every padding float of the blob and the moments are never written.  activation WL_ACTIVATION_ELU:
 * obs_dim 1..16; WL_ACTIVATION_RELU: obs_dim 1..4096.  One call enqueues the whole update, never syncs the host and is
 * graph-capturable; no float atomics, so results are bit-identical run to run for a given (N, gradient_length, SM count).
 * d_state[wl_distill_state_floats(T, num_learning_epochs)] (fp32; the caller sets [0] = learning rate, [1] = 0):
 *   [0] learning rate  [1] Adam step count  [2] the mean of this update's per-step losses (rsl_rl's Loss/behavior)
 *   [3] the number of Adam steps this update took  [4 + i] the loss of the i-th step walked (i < T * epochs)
 * Bad arguments (T < gradient_length, ELU with obs_dim > 16, a null or misaligned pointer, a short workspace) return
 * WL_EINVAL / WL_EUNSUPPORTED before any launch. */
typedef struct wl_distill_params {
    int32_t obs_dim;                /* the student's input width */
    int32_t num_learning_epochs;
    int32_t gradient_length;        /* stored steps per Adam step */
    float max_grad_norm;            /* > 0: clip the actor's gradient norm; <= 0: no clip (rsl_rl's None) */
} wl_distill_params;
int32_t wl_distill_state_floats(int32_t T, int32_t num_learning_epochs);
/* workspace for wl_distill_update on the current device (0 and wl_last_error() on error) */
size_t wl_distill_workspace_bytes(int32_t obs_dim, int32_t n_envs, int32_t gradient_length);
int wl_distill_update(const wl_distill_params* params, const float* d_obs, const float* d_teacher_actions, int32_t T, int32_t N,
                      int32_t activation, float* d_blob, float* d_adam_m, float* d_adam_v, float* d_state, void* d_workspace,
                      size_t workspace_bytes, void* stream);

/* ---- the wide asymmetric actor-critic: a critic input of its own (DESIGN.md 6s) ------------------------------------------
 * The network above with the critic's first layer fed from a second row, d_critic_obs_in [N, critic_obs_dim], and a blob
 * laid out by wl_policy_blob_floats_asym(obs_dim, critic_obs_dim); obs_dim and critic_obs_dim in 1..4096.
 * Each net's layer 1 keeps wl_policy_act's K chunks (32 inputs from 0, each summed alone, then added to the running sum
 * from the bias); a net that has run out of chunks adds nothing.  So actions, mean and log-prob equal wl_policy_act's for
 * the same d_obs_in and actor blocks bit for bit whatever the critic input is, and with critic_obs_dim == obs_dim and
 * d_critic_obs_in == d_obs_in the value does too.  Returns before any launch as wl_policy_act does, plus WL_EINVAL for a
 * null / misaligned d_critic_obs_in or critic_obs_dim outside 1..4096. */
int wl_policy_act_wide_asym(wl_sim* sim, const float* d_obs_in, const float* d_critic_obs_in, int32_t critic_obs_dim,
                            const float* d_policy_blob, wl_policy_out out, int64_t step_counter, void* stream);
/* wl_ppo_update_wide for that network: the critic's layer-1 forward and its dW1 are taken over d_critic_obs [batch,
 * critic_obs_dim] (slab order, gathered through the same perm); the layers 2-3 kernel is wl_ppo_update_wide's; the
 * reduction and Adam step skip the padding rows of both W1t blocks.  No float atomics, a fixed sum order.  With
 * critic_obs_dim == obs_dim and d_critic_obs == batch->obs it leaves blob, moments and state equal to wl_ppo_update_wide's,
 * bit for bit.  d_critic_obs 4-byte aligned; otherwise wl_ppo_update_wide's checks. */
size_t wl_ppo_wide_asym_workspace_bytes(int32_t obs_dim, int32_t critic_obs_dim, int32_t batch, int32_t num_mini_batches);
int wl_ppo_update_wide_asym(const wl_ppo_params* params, const wl_ppo_batch* batch, const float* d_critic_obs, int32_t critic_obs_dim,
                            float* d_blob, float* d_adam_m, float* d_adam_v, float* d_state, void* d_workspace, size_t workspace_bytes,
                            void* stream);

/* ---- the data-parallel PPO update: rsl_rl's multi-GPU PPO.update() [UPSTREAM-RECALL] ------------------------------------
 * n_ranks replicas of the update above (activation WL_ACTIVATION_ELU: wl_ppo_update's network; WL_ACTIVATION_RELU:
 * wl_ppo_update_wide's), each on its own rows, with the gradient and the KL averaged across the ranks inside every
 * mini-batch: each rank's reduced gradient (entropy term included) and kl_mean are summed in rank order 0..n_ranks-1 and
 * divided by n_ranks, then the KL rule, clip_grad_norm_ and Adam run on the average, so every replica forms the same bits.
 * Rank-local as in the single-rank update: advantage normalisation, the permutation, the loss statistics in d_state.
 * d_exchange[r] (r < n_ranks, 256-byte aligned) = rank r's exchange buffer of wl_ppo_dp_exchange_bytes(obs_dim) bytes, the
 * same rank order on every rank: this process's own buffers and the P2P-mapped buffers of its peers (e.g. one torch
 * symmetric-memory allocation), zero-filled once before the first call and left to the calls afterwards.  The call runs
 * n_local ranks, local_ranks[l] being the rank of the l-th entry of the per-rank arrays (batches, d_blob, d_adam_m,
 * d_adam_v, d_state, d_workspace: wl_ppo_update's arguments, one per local rank; workspace_bytes as wl_ppo_workspace_bytes /
 * wl_ppo_wide_workspace_bytes); their exchange buffers must be on one device.  One local rank per process is the
 * multi-process form; all ranks local (one device, one stream) runs the whole exchange in one process.  Each mini-batch
 * waits on the device for every peer's row (no host sync, graph-capturable: the round counter lives in the buffers); a
 * wait that exceeds 60 s sets word 1 of the rank's own buffer (uint32, nonzero = failed), after which the call leaves
 * blob, moments and d_state untouched.  n_ranks = 1 gives wl_ppo_update / wl_ppo_update_wide's results bit for bit.
 * Bad arguments (n_ranks outside 1..WL_MAX_PEERS, a null or misaligned exchange buffer, a local rank index out of range or
 * repeated, local buffers on different devices, and every argument error of the single-rank entries) return WL_EINVAL
 * before any launch. */
size_t wl_ppo_dp_exchange_bytes(int32_t obs_dim);
int wl_ppo_update_dp(const wl_ppo_params* params, int32_t activation, int32_t n_ranks, void* const* d_exchange, int32_t n_local,
                     const int32_t* local_ranks, const wl_ppo_batch* batches, float* const* d_blob, float* const* d_adam_m,
                     float* const* d_adam_v, float* const* d_state, void* const* d_workspace, size_t workspace_bytes, void* stream);

/* A caller that drives wl_step through a CUDA graph of K steps (how a rollout is meant to be issued: one launch per K steps)
 * pays the upload of the instantiated graph to the device on its FIRST launch; this moves that
 * upload to set-up time.  graph_exec = cudaGraphExec_t (torch: CUDAGraph.raw_cuda_graph_exec()). */
int wl_graph_upload(void* graph_exec, void* stream);

/* ---- test hooks (bit-exactness of the deterministic math vs the oracle) ------ */
/* op: 0 sin,1 cos,2 atan,3 atan2(x=in,y=in2),4 log,5 tan,6 asin,7 exp,8 tanh ; out[n] */
int wl_test_detmath(int32_t op, const float* d_in, const float* d_in2, float* d_out, int32_t n,
                    void* stream);
/* an empty kernel of the given geometry (launch / event-timing floor of the measurement protocol) */
int wl_test_null(int32_t grid, int32_t block, void* stream);
int wl_test_null_cfg(wl_sim* sim, int32_t grid, int32_t block, void* stream);   /* same, with the wl_config kernel parameter */
/* philox4x32-10: out[4*n] for counters (c0_base + i, c1, c2, c3), key from seed */
int wl_test_philox(uint64_t seed, uint32_t c0_base, uint32_t c1, uint32_t c2, uint32_t c3, uint32_t* d_out,
                   int32_t n, void* stream);
/* the handle's device-term kernels (wl_terms_kernel, and wl_terms_log_kernel when d_term_log is not NULL) on a caller-given
 * state: d_state in the handle's [group][N] float4 layout (the pre-reset state wl_step_stage_a leaves), d_done[N] the
 * built-in termination bytes (nonzero: done), d_rew[N] in / out (the reward terms are added to it), d_term_log as in
 * wl_step_terms.  It reads and updates the handle's term state (episode sums, previous elevations, the fired bits of
 * wl_device_term_masks) exactly as wl_step_terms does; the handle's own state buffer is not touched.  WL_EINVAL for a null
 * argument, a state that is not 16-byte aligned, a negative step counter or a handle without device terms. */
int wl_test_device_terms(wl_sim* sim, const float* d_state, const uint8_t* d_done, float* d_rew, float* d_term_log,
                         int64_t step_counter, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* WHEELEDLAB_B200_H */
