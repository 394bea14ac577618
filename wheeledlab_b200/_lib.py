"""ctypes binding of the C-ABI in ``include/wheeledlab_b200.h``.

The CUDA library is the ONLY compute path of this package: if it is missing, importing
this module raises (there is no CPU / eager fallback by design).
"""
from __future__ import annotations

import ctypes as C
import os
from pathlib import Path

_PKG_DIR = Path(__file__).resolve().parent
LIB_PATH = Path(os.environ["WHEELEDLAB_B200_LIB"]) if os.environ.get("WHEELEDLAB_B200_LIB") else _PKG_DIR / "libwheeledlab_b200.so"   # (override: kernel A/B builds)

_TAGS = {"i32": C.c_int32, "u64": C.c_uint64, "f32": C.c_float}


class NativeLibraryMissing(ImportError):
    pass


def _load() -> C.CDLL:
    if not LIB_PATH.exists():
        raise NativeLibraryMissing(
            f"{LIB_PATH} not found. wheeledlab_b200 has no CPU fallback: build the sm_90a extension first "
            f"(python -c 'import __graft_entry__ as g; g.build()' from the repo root)."
        )
    return C.CDLL(str(LIB_PATH), mode=os.RTLD_GLOBAL if hasattr(os, "RTLD_GLOBAL") else C.DEFAULT_MODE)


lib = _load()

lib.wl_config_describe.restype = C.c_char_p
lib.wl_config_sizeof.restype = C.c_size_t
lib.wl_last_error.restype = C.c_char_p
lib.wl_build_info.restype = C.c_char_p


def make_config_struct(describe: str, name: str = "WlConfig"):
    """Build a ctypes.Structure from a ``wl_config_describe()`` string and verify offsets."""
    fields, offsets, size = [], {}, None
    for item in describe.split(";"):
        if not item:
            continue
        parts = item.split(":")
        if parts[0] == "sizeof":
            size = int(parts[1])
            continue
        fname, tag, count, off = parts[0], parts[1], int(parts[2]), int(parts[3])
        ctype = _TAGS[tag]
        fields.append((fname, ctype if count == 1 else ctype * count))
        offsets[fname] = off
    cls = type(name, (C.Structure,), {"_fields_": fields})
    for fname, off in offsets.items():
        got = getattr(cls, fname).offset
        if got != off:
            raise RuntimeError(f"wl_config layout mismatch at {fname}: ctypes {got} vs C {off}")
    if size is not None and C.sizeof(cls) != size:
        raise RuntimeError(f"wl_config size mismatch: ctypes {C.sizeof(cls)} vs C {size}")
    return cls


CONFIG_DESCRIBE = lib.wl_config_describe().decode()
WlConfig = make_config_struct(CONFIG_DESCRIBE)


class WlGlobals(C.Structure):
    _fields_ = [
        ("rew_weight", (C.c_float * 8) * 2),
        ("acc", (C.c_float * 16) * 3),
        ("log_ptr", C.c_void_p * 3),
        ("last_log", C.c_float * 16),
        ("step_base", C.c_uint32),
        ("ticket", C.c_uint32),
        ("curr_applied_t", C.c_uint32),
        ("_pad", C.c_uint32 * 1),
    ]


_vp, _i32, _i64, _u32, _u64, _sz = C.c_void_p, C.c_int32, C.c_int64, C.c_uint32, C.c_uint64, C.c_size_t
lib.wl_config_finalize.argtypes = [C.POINTER(WlConfig)]
lib.wl_set_step_counter.argtypes = [_vp, _i64, _vp]
lib.wl_set_seed.argtypes = [_vp, _u64]
lib.wl_set_term_bits.argtypes = [_vp, _vp]
lib.wl_set_peer_fanout.argtypes = [_vp, _i32, C.POINTER(_i64)]
lib.wl_set_multicast_fanout.argtypes = [_vp, C.c_int64]
lib.wl_advance_counter.argtypes = [_vp, _i32, _vp]
lib.wl_note_device_counter.argtypes = [_vp, _i64]
lib.wl_log_flush.argtypes = [_vp, _vp]
lib.wl_reward_weights.restype = _vp
lib.wl_reward_weights.argtypes = [_vp]
lib.wl_state_bytes.restype = _sz
lib.wl_state_bytes.argtypes = [_i32]
lib.wl_globals_offset.restype = _sz
lib.wl_globals_offset.argtypes = [_i32]
lib.wl_create.argtypes = [C.POINTER(WlConfig), _vp, _sz, _vp, C.POINTER(_vp)]
lib.wl_destroy.argtypes = [_vp]
lib.wl_startup.argtypes = [_vp, _vp]
lib.wl_reset.argtypes = [_vp, _vp, _i32, _i64, _vp]
lib.wl_step.argtypes = [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _i64, _vp]
lib.wl_observe.argtypes = [_vp, _vp, _i64, _i32, _vp]
lib.wl_rollout.argtypes = [_vp, _i32, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i64, _vp]
lib.wl_result_bytes.restype = _sz
lib.wl_result_bytes.argtypes = [_i32]
lib.wl_step_host.argtypes = [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i64, _vp]
lib.wl_step_host_zero_copy.argtypes = [_vp, _vp, _vp, _vp, _vp, _i64, _vp]
lib.wl_curriculum.argtypes = [_vp, _i32, C.POINTER(_i32), C.POINTER(C.c_float), _u32, _vp]
lib.wl_synth_actions.argtypes = [_vp, _vp, _i64, _i32, _vp]
lib.wl_derive_suspension.argtypes = [_vp, _vp, _vp, _vp]
lib.wl_set_kernel_variant.argtypes = [_vp, _i32]
lib.wl_set_scan_tma.argtypes = [_vp, _i32]
lib.wl_obs_dim.restype = _i32
lib.wl_obs_dim.argtypes = [_vp]
lib.wl_launch_count.restype = _i64
lib.wl_launch_count.argtypes = [_vp]
lib.wl_chained_step_count.restype = _i64
lib.wl_chained_step_count.argtypes = [_vp]
lib.wl_deep_step_count.restype = _i64
lib.wl_deep_step_count.argtypes = [_vp]
lib.wl_step_launch_info.argtypes = [_vp, C.POINTER(_i32), C.POINTER(_u32), C.POINTER(_i32), C.POINTER(_i32)]


class WlPolicyOut(C.Structure):
    _fields_ = [("actions", _vp), ("mean", _vp), ("log_prob", _vp), ("value", _vp)]


lib.wl_policy_blob_floats.restype = _i32
lib.wl_policy_blob_floats.argtypes = [_i32, C.POINTER(_i32)]
lib.wl_act_step.argtypes = [_vp, _vp, _vp, WlPolicyOut, _vp, _vp, _vp, _vp, _vp, _i64, _vp]
lib.wl_policy_act.argtypes = [_vp, _vp, _vp, WlPolicyOut, _i64, _vp]
lib.wl_act_infer_step.argtypes = [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i64, _vp]
lib.wl_policy_act_elu.argtypes = [_vp, _vp, _vp, WlPolicyOut, _i64, _vp]
lib.wl_actor_mean.argtypes = [_vp, _i32, _i32, _vp, _i32, _vp, _vp]
WL_ACTIVATION = {"elu": 0, "relu": 1}       # WL_ACTIVATION_ELU / WL_ACTIVATION_RELU
lib.wl_camera.argtypes = [_vp, _vp, _i64, _vp, _vp]
lib.wl_step_stage_a.argtypes = [_vp, _vp, _vp, _vp, _i64, _vp]
lib.wl_step_stage_b.argtypes = [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i64, _vp]
lib.wl_step_stage_b1.argtypes = [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _i64, _vp]
lib.wl_step_stage_b2.argtypes = [_vp, _vp, _i64, _vp]
WL_MAX_EVENT_TERMS = 8
lib.wl_set_event_timers.argtypes = [_vp, _i32, _vp]
lib.wl_event_timers.argtypes = [_vp, _vp, _vp, _i64, _vp]


class WlTermDesc(C.Structure):
    _fields_ = [("kind", _i32), ("role", _i32), ("weight", C.c_double), ("params", C.c_double * 4)]


lib.wl_set_device_terms.argtypes = [_vp, _vp, _i32]
lib.wl_step_terms.argtypes = [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i64, _vp]
lib.wl_device_term_masks.restype = _vp
lib.wl_device_term_masks.argtypes = [_vp]


class WlDeviceEventDesc(C.Structure):
    _fields_ = [("mode", _i32), ("interval_range_s", C.c_float * 2), ("velocity_range", (C.c_float * 2) * 6)]


WL_MAX_DEVICE_EVENTS = 8
WL_EVENT_MODE = {"reset": 1, "interval": 2}   # WL_EVENT_MODE_RESET / _INTERVAL
lib.wl_set_device_events.argtypes = [_vp, _vp, _i32]
lib.wl_device_events.argtypes = [_vp, _vp, _vp, _i64, _vp]


class WlCriticTerm(C.Structure):
    _fields_ = [("kind", _i32), ("clip", C.c_float)]


# WL_CRITIC_*: the critic observation's term library (name -> kind, width)
WL_CRITIC_TERMS = {"root_pos_w": (1, 3), "root_euler_xyz": (2, 3), "base_lin_vel": (3, 3), "base_ang_vel": (4, 3), "last_action": (5, 2),
                   "joint_vel": (6, 4), "joint_pos": (7, 2), "wheel_friction": (8, 4), "base_mass": (9, 1), "motor_damping": (10, 4)}
WL_MAX_CRITIC_OBS = 32
lib.wl_set_critic_terms.argtypes = [_vp, _vp, _i32]
lib.wl_critic_obs_dim.restype = _i32
lib.wl_critic_obs_dim.argtypes = [_vp]
lib.wl_critic_observe.argtypes = [_vp, _vp, _vp]


class WlPolicyTerm(C.Structure):
    _fields_ = [("kind", _i32), ("noise", _i32), ("noise_params", C.c_double * 2), ("clip", _i32), ("n_scale", _i32),
                ("clip_range", C.c_double * 2), ("scale", C.c_double * 4)]


# WL_POLICY_*: the policy observation's term library (name -> kind, width): the critic library and projected_gravity
WL_POLICY_TERMS = dict(WL_CRITIC_TERMS, projected_gravity=(11, 3))
WL_MAX_POLICY_OBS = 32
WL_NOISE = {None: 0, "gaussian": 1, "uniform": 2}
WL_POLICY_OBS_AFTER_STEP = -1
lib.wl_set_policy_terms.argtypes = [_vp, _vp, _i32]
lib.wl_policy_obs_dim.restype = _i32
lib.wl_policy_obs_dim.argtypes = [_vp]
lib.wl_policy_observe.argtypes = [_vp, _i64, _i32, _vp, _vp]
# WL_ROW_*: the terms of the Elevation / Visual built-in rows (name -> kind, width), and each task's row in order
WL_ROW_TERMS = {"goal_relative_xyz": (12, 2), "root_euler_xyz": (2, 3), "base_lin_vel": (3, 3), "base_ang_vel": (4, 3),
                "last_action": (5, 2), "world_height_map": (13, 676)}
WL_ROW_TASK_TERMS = {"elevation": ("goal_relative_xyz", "root_euler_xyz", "base_lin_vel", "base_ang_vel", "last_action", "world_height_map"),
                     "visual": ("base_lin_vel", "base_ang_vel", "last_action")}
lib.wl_set_row_terms.argtypes = [_vp, _vp, _i32]
lib.wl_row_terms.restype = _i32
lib.wl_row_terms.argtypes = [_vp]
lib.wl_set_row_critic.argtypes = [_vp, _vp, _i32, _vp, _i32]
# WL_RESET_EV_*: the DR events wl_set_reset_events can redraw at every reset (name -> bit)
WL_RESET_EVENTS = {"material": 1, "actuator_gains": 2, "base_mass": 4, "wheel_mass": 8}
lib.wl_set_reset_events.argtypes = [_vp, _u32]
lib.wl_reset_events.restype = _u32
lib.wl_reset_events.argtypes = [_vp]
lib.wl_policy_blob_floats_asym.restype = _i32
lib.wl_policy_blob_floats_asym.argtypes = [_i32, _i32, C.POINTER(_i32)]
lib.wl_policy_act_asym.argtypes = [_vp, _vp, _vp, _i32, _vp, WlPolicyOut, _i64, _vp]
lib.wl_gae.argtypes = [_vp, _vp, _vp, _vp, _vp, C.c_float, C.c_float, _vp, _vp, _i32, _i32, _vp]


class WlEpisodeStatsState(C.Structure):
    _fields_ = [("ring_return", C.c_float * 100), ("ring_length", C.c_float * 100), ("fill", _i32), ("head", _i32),
                ("finished", _i32), ("_pad", _i32), ("mean_return", C.c_double), ("mean_length", C.c_double)]


lib.wl_episode_stats_workspace_bytes.restype = _sz
lib.wl_episode_stats_workspace_bytes.argtypes = [_i32, _i32]
lib.wl_episode_stats.argtypes = [_vp, _vp, _vp, _i32, _i32, _vp, _vp, _vp, _vp, _sz, _vp]
lib.wl_dp_adam_step.argtypes = [_vp, _vp, _vp, _i32, C.POINTER(_vp), C.c_float, C.c_double, C.c_double, C.c_float, C.c_float, _i32, _i32, _vp]


class WlPpoParams(C.Structure):
    _fields_ = [("obs_dim", _i32), ("batch", _i32), ("num_learning_epochs", _i32), ("num_mini_batches", _i32),
                ("clip_param", C.c_float), ("value_loss_coef", C.c_float), ("entropy_coef", C.c_float),
                ("max_grad_norm", C.c_float), ("desired_kl", C.c_float), ("adaptive", _i32),
                ("use_clipped_value_loss", _i32), ("_pad", _i32)]


class WlPpoBatch(C.Structure):
    _fields_ = [("obs", _vp), ("actions", _vp), ("values", _vp), ("log_prob", _vp), ("mean", _vp), ("returns", _vp),
                ("advantages", _vp), ("perm", _vp)]


lib.wl_ppo_state_floats.restype = _i32
lib.wl_ppo_state_floats.argtypes = []
lib.wl_ppo_workspace_bytes.restype = _sz
lib.wl_ppo_workspace_bytes.argtypes = [_i32, _i32, _i32]
lib.wl_ppo_update.argtypes = [C.POINTER(WlPpoParams), C.POINTER(WlPpoBatch), _vp, _vp, _vp, _vp, _vp, _sz, _vp]
lib.wl_ppo_asym_workspace_bytes.restype = _sz
lib.wl_ppo_asym_workspace_bytes.argtypes = [_i32, _i32, _i32, _i32]
lib.wl_ppo_update_asym.argtypes = [C.POINTER(WlPpoParams), C.POINTER(WlPpoBatch), _vp, _i32, _vp, _vp, _vp, _vp, _vp, _sz, _vp]
lib.wl_ppo_wide_workspace_bytes.restype = _sz
lib.wl_ppo_wide_workspace_bytes.argtypes = [_i32, _i32, _i32]
lib.wl_ppo_update_wide.argtypes = [C.POINTER(WlPpoParams), C.POINTER(WlPpoBatch), _vp, _vp, _vp, _vp, _vp, _sz, _vp]
lib.wl_policy_act_wide_asym.argtypes = [_vp, _vp, _vp, _i32, _vp, WlPolicyOut, _i64, _vp]
lib.wl_ppo_wide_asym_workspace_bytes.restype = _sz
lib.wl_ppo_wide_asym_workspace_bytes.argtypes = [_i32, _i32, _i32, _i32]
lib.wl_ppo_update_wide_asym.argtypes = [C.POINTER(WlPpoParams), C.POINTER(WlPpoBatch), _vp, _i32, _vp, _vp, _vp, _vp, _vp, _sz, _vp]
lib.wl_ppo_dp_exchange_bytes.restype = _sz
lib.wl_ppo_dp_exchange_bytes.argtypes = [_i32]
lib.wl_ppo_update_dp.argtypes = [C.POINTER(WlPpoParams), _i32, _i32, C.POINTER(_vp), _i32, C.POINTER(_i32), C.POINTER(WlPpoBatch),
                                 C.POINTER(_vp), C.POINTER(_vp), C.POINTER(_vp), C.POINTER(_vp), C.POINTER(_vp), _sz, _vp]


class WlDistillParams(C.Structure):
    _fields_ = [("obs_dim", _i32), ("num_learning_epochs", _i32), ("gradient_length", _i32), ("max_grad_norm", C.c_float)]


lib.wl_distill_state_floats.restype = _i32
lib.wl_distill_state_floats.argtypes = [_i32, _i32]
lib.wl_distill_workspace_bytes.restype = _sz
lib.wl_distill_workspace_bytes.argtypes = [_i32, _i32, _i32]
lib.wl_distill_update.argtypes = [C.POINTER(WlDistillParams), _vp, _vp, _i32, _i32, _i32, _vp, _vp, _vp, _vp, _vp, _sz, _vp]
lib.wl_test_detmath.argtypes = [_i32, _vp, _vp, _vp, _i32, _vp]
lib.wl_test_philox.argtypes = [_u64, _u32, _u32, _u32, _u32, _vp, _i32, _vp]
lib.wl_test_device_terms.argtypes = [_vp, _vp, _vp, _vp, _vp, _i64, _vp]
lib.wl_test_null.argtypes = [_i32, _i32, _vp]
lib.wl_test_null_cfg.argtypes = [_vp, _i32, _i32, _vp]
lib.wl_graph_upload.argtypes = [_vp, _vp]

EXPORTED_SYMBOLS = [
    "wl_config_describe", "wl_config_sizeof", "wl_config_finalize", "wl_set_step_counter", "wl_advance_counter", "wl_note_device_counter", "wl_log_flush", "wl_reward_weights", "wl_set_seed", "wl_set_term_bits", "wl_set_peer_fanout", "wl_set_multicast_fanout", "wl_state_bytes", "wl_globals_offset", "wl_create", "wl_destroy",
    "wl_last_error", "wl_build_info", "wl_startup", "wl_reset", "wl_step", "wl_step_host", "wl_step_host_zero_copy", "wl_rollout", "wl_result_bytes", "wl_observe", "wl_curriculum",
    "wl_synth_actions", "wl_derive_suspension", "wl_set_kernel_variant", "wl_set_scan_tma", "wl_obs_dim", "wl_launch_count", "wl_chained_step_count", "wl_deep_step_count", "wl_step_launch_info", "wl_policy_blob_floats", "wl_act_step", "wl_step_stage_a", "wl_step_stage_b", "wl_step_stage_b1", "wl_step_stage_b2", "wl_set_event_timers", "wl_event_timers", "wl_set_device_terms", "wl_step_terms", "wl_device_term_masks", "wl_set_device_events", "wl_device_events", "wl_camera", "wl_gae", "wl_dp_adam_step", "wl_ppo_state_floats", "wl_ppo_workspace_bytes", "wl_ppo_update", "wl_policy_act", "wl_ppo_wide_workspace_bytes", "wl_ppo_update_wide", "wl_ppo_dp_exchange_bytes", "wl_ppo_update_dp", "wl_episode_stats_workspace_bytes", "wl_episode_stats", "wl_act_infer_step", "wl_policy_act_elu", "wl_actor_mean", "wl_set_critic_terms", "wl_critic_obs_dim", "wl_critic_observe", "wl_set_policy_terms", "wl_policy_obs_dim", "wl_policy_observe", "wl_set_row_terms", "wl_row_terms", "wl_set_reset_events", "wl_reset_events", "wl_policy_blob_floats_asym", "wl_policy_act_asym", "wl_ppo_asym_workspace_bytes", "wl_ppo_update_asym", "wl_set_row_critic", "wl_policy_act_wide_asym", "wl_ppo_wide_asym_workspace_bytes", "wl_ppo_update_wide_asym", "wl_distill_state_floats", "wl_distill_workspace_bytes", "wl_distill_update", "wl_graph_upload", "wl_test_detmath", "wl_test_philox", "wl_test_device_terms", "wl_test_null", "wl_test_null_cfg",
]


class WlError(RuntimeError):
    pass


def check(rc: int, what: str = "") -> None:
    if rc != 0:
        raise WlError(f"{what} failed (code {rc}): {lib.wl_last_error().decode()}")
