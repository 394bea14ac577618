"""The row terms' CPU twin (tests/row_terms_oracle.c, DESIGN 6r): TEST INFRASTRUCTURE ONLY.

The C file includes the unchanged oracle and adds wlo_row_observe / wlo_row_raw / wlo_row_draw; it is compiled, with the
oracle's own flags, into a temporary directory on first use (the source tree may be read-only).  ``RowOracle`` is an
``oracle_lib.Oracle`` on that library (start-up, reset, step, observe, state import / export), which also forms the rows
under row terms.  Row terms are a list of (name, noise, clip, scale) as ``WheeledSim.set_row_terms`` takes them."""
from __future__ import annotations

import atexit
import ctypes as C
import os
import shutil
import subprocess
import tempfile
from pathlib import Path

import numpy as np

import oracle_lib as O

HERE = Path(__file__).resolve().parent
_LIB = None
NOISE = {None: 0, "gaussian": 1, "uniform": 2}
# the terms of the Elevation / Visual rows (WL_ROW_GOAL_RELATIVE_XYZ, WL_CRITIC_*, WL_ROW_WORLD_HEIGHT_MAP): name -> (kind, width)
ROW_KINDS = {"goal_relative_xyz": (12, 2), "root_euler_xyz": (2, 3), "base_lin_vel": (3, 3), "base_ang_vel": (4, 3), "last_action": (5, 2),
             "world_height_map": (13, 676)}


def get_lib():
    global _LIB
    if _LIB is None:
        out = Path(tempfile.mkdtemp(prefix="wl_row_terms_oracle_"))
        atexit.register(shutil.rmtree, out, True)
        fma = ["-mfma"] if " fma " in Path("/proc/cpuinfo").read_text().replace("\n", " ") else []
        cc = os.environ.get("WLO_CC", "/usr/bin/gcc")
        so = out / "libwl_row_terms_oracle.so"
        subprocess.run([cc, "-O2", "-std=c11", *fma, "-fPIC", "-shared", "-ffp-contract=off", "-fno-fast-math", "-fopenmp",
                        "-o", str(so), str(HERE / "row_terms_oracle.c"), "-lm"], check=True)
        lib = C.CDLL(str(so))
        vp, i32, i64, u32, u64 = C.c_void_p, C.c_int32, C.c_int64, C.c_uint32, C.c_uint64
        # the oracle's entry points RowOracle uses, declared as oracle_lib declares them
        lib.wlo_create.restype = vp
        lib.wlo_create.argtypes = [vp, vp]
        lib.wlo_destroy.argtypes = [vp]
        lib.wlo_startup.argtypes = [vp]
        lib.wlo_reset.argtypes = [vp, vp, i32, i64]
        lib.wlo_step.argtypes = [vp, vp, vp, vp, vp, vp, i64, i32]
        lib.wlo_observe.argtypes = [vp, vp, i64, i32]
        lib.wlo_export_state.argtypes = [vp, vp]
        lib.wlo_import_state.argtypes = [vp, vp]
        lib.wlo_row_observe.argtypes = [vp, vp, i32, i64, i32, vp]
        lib.wlo_row_raw.argtypes = [vp, vp]
        lib.wlo_row_draw.argtypes = [u64, u32, u32, i32, i32, i32]
        lib.wlo_row_draw.restype = C.c_float
        _LIB = lib
    return _LIB


class PolicyTerm(C.Structure):
    """wl_policy_term"""
    _fields_ = [("kind", C.c_int32), ("noise", C.c_int32), ("noise_params", C.c_double * 2), ("clip", C.c_int32), ("n_scale", C.c_int32),
                ("clip_range", C.c_double * 2), ("scale", C.c_double * 4)]


def row_table(terms):
    """A wl_policy_term array from (name, noise, clip, scale) rows (noise None / (kind, a, b); scale None, a number or a tuple)."""
    arr = (PolicyTerm * max(1, len(terms)))()
    for k, (name, noise, clip, scale) in enumerate(terms):
        d = arr[k]
        d.kind = ROW_KINDS[name][0]
        if noise is not None:
            d.noise = NOISE[noise[0]]
            d.noise_params[0], d.noise_params[1] = float(noise[1]), float(noise[2])
        if clip is not None:
            d.clip = 1
            d.clip_range[0], d.clip_range[1] = float(clip[0]), float(clip[1])
        if scale is not None:
            sc = (float(scale),) if isinstance(scale, (int, float)) else tuple(float(s) for s in scale)
            d.n_scale = len(sc)
            for j, s in enumerate(sc):
                d.scale[j] = s
    return arr


def row_draw(seed, gid, t, call_idx, j, kind) -> np.float32:
    """wlo_row_draw: the row-terms noise draw of row column j, z (kind "gaussian") or u in [0, 1) (kind "uniform")."""
    return np.float32(get_lib().wlo_row_draw(seed, gid, t & 0xFFFFFFFF, call_idx, j, NOISE[kind]))


class RowOracle(O.Oracle):
    """oracle_lib.Oracle on the twin's library (the unchanged oracle plus the row-terms entries)."""

    def __init__(self, cfg, heightfield=None, threads=1):
        self.lib = get_lib()
        self.cfg = cfg
        self.n = int(cfg.num_envs)
        self.threads = threads
        self.obs_dim = {0: 14, 1: 689, 2: 8}[int(cfg.task)]
        if int(cfg.task) == 2 and int(cfg.vis_cam):
            self.obs_dim += int(cfg.vis_cam_w) * (int(cfg.vis_cam_h) - int(cfg.vis_cam_row0))
        if heightfield is None:
            hf = None
        elif int(cfg.task) == 2:
            hf = np.ascontiguousarray(heightfield)                      # raw aux bytes (visual)
        else:
            hf = np.ascontiguousarray(heightfield, dtype=np.float32)
        self._hf = hf
        self._h = C.c_void_p(self.lib.wlo_create(C.byref(cfg), O._p(hf)))

    def row_observe(self, terms, step_counter, call_idx=-1, obs=None):
        """wlo_row_observe: the row of every env under the row terms (name, noise, clip, scale), written into `obs` [N,
        obs_dim] (a new zeroed array when None; on Visual only the 8 tail floats are written)."""
        obs = np.zeros((self.n, self.obs_dim), np.float32) if obs is None else obs
        assert obs.dtype == np.float32 and obs.shape == (self.n, self.obs_dim) and obs.flags.c_contiguous
        assert self.lib.wlo_row_observe(self._h, row_table(terms), len(terms), step_counter, call_idx, O._p(obs)) == 0
        return obs

    def row_raw(self):
        """wlo_row_raw: the raw row columns [N, 689] (Elevation) or [N, 8] (Visual tail) of the current state."""
        raw = np.empty((self.n, 8 if int(self.cfg.task) == 2 else 689), np.float32)
        assert self.lib.wlo_row_raw(self._h, O._p(raw)) == 0
        return raw
