"""The device-term golden fixture (tests/golden/device_terms.npz, written by make_golden.py from the reference's own
functions) as oracle / kernel inputs: the config, the state array in the product's [group][N] float4 layout, and one
term table per (function, parameter set).  Shared by test_device_terms_oracle_cpu.py and test_device_terms_edges_gpu.py."""
from __future__ import annotations

from pathlib import Path

import numpy as np

G = np.load(Path(__file__).resolve().parent / "golden" / "device_terms.npz")
NUM_GROUPS = 16
G_POS, G_QUAT, G_LINVEL, G_ANGVEL, G_WHEEL = range(5)
ROLE_REWARD, ROLE_TERMINATION, ROLE_TIME_OUT = 0, 1, 2
KINDS = {"forward_vel": 1, "forward_wheel_spin": 2, "change_in_elevation": 3, "ascending": 4, "steep_penalty": 5,
         "elevation_continuity": 6, "yaw_change_onElev": 7, "upright_penalty": 8, "roll_on_elev": 9, "low_vel_penalty": 10,
         "is_traversable": 11, "is_traversable_speed_scaled": 12, "vel_rew_trav": 13, "low_speed_penalty": 14, "off_track": 15,
         "bool_is_not_traversable": 16, "roll_over": 17}
# the functions of one state each (elevation_continuity has its own sequences; bool_is_not_traversable its own counters)
STATE_FUNCS = [k for k in KINDS if k not in ("elevation_continuity", "bool_is_not_traversable")]
N = int(G["pos"].shape[0])


def config(n=N):
    """The Visual task's config over the golden's map (map terms need the Visual task; the others read only the state)."""
    import wheeledlab_b200 as wl
    spec = wl.visual_task(num_envs=n, seed=1, traversability=G["map"].astype(bool))
    assert int(spec.cfg.max_episode_length) == int(G["max_episode_length"])
    assert float(spec.cfg.vis_row_spacing) == float(G["spacing"]) == float(spec.cfg.vis_col_spacing)
    return spec


def step_dt(cfg):
    return float(cfg.sim_dt) * int(cfg.decimation)


def state(pos=None, z=None):
    """[16, N, 4] float32: the golden's states (or pos.z replaced by z)."""
    p = G["pos"] if pos is None else pos
    n = p.shape[0]
    st = np.zeros((NUM_GROUPS, n, 4), np.float32)
    st[G_POS, :, :3] = p
    if z is not None:
        st[G_POS, :, 2] = z
    if pos is None:
        st[G_QUAT] = G["quat"]
        st[G_LINVEL, :, :3] = G["vel_w"]
        st[G_ANGVEL, :, :3] = G["ang_w"]
        st[G_WHEEL] = G["omega"]
    else:
        st[G_QUAT, :, 0] = 1.0
    return st


def table(name, params, cfg, role=ROLE_REWARD):
    """One term: a reward of weight 1 / step_dt (fp32(weight * step_dt) = 1, so the reward is the value) or a termination."""
    w = 1.0 / step_dt(cfg) if role == ROLE_REWARD else 0.0
    return [(KINDS[name], role, w, list(params))]
