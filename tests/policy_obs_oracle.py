"""The policy observation table's CPU twin (tests/policy_obs_oracle.c): TEST INFRASTRUCTURE ONLY.

The C file is compiled, with the oracle's own flags, into a temporary directory on first use (the source tree may be
read-only).  A table is a list of (library name, noise, clip, scale) as ``WheeledSim.set_policy_terms`` takes it; the
state is the device state's groups, float32 [WL_NUM_GROUPS, N, 4] (``sim.groups``)."""
from __future__ import annotations

import atexit
import ctypes as C
import os
import shutil
import subprocess
import tempfile
from pathlib import Path

import numpy as np

HERE = Path(__file__).resolve().parent
_LIB = None
# first library float and width of each term (the row the kernel forms per env: the critic library, then gravity)
LIBRARY = {"root_pos_w": (0, 3), "root_euler_xyz": (3, 3), "base_lin_vel": (6, 3), "base_ang_vel": (9, 3), "last_action": (12, 2),
           "joint_vel": (14, 4), "joint_pos": (18, 2), "wheel_friction": (20, 4), "base_mass": (24, 1), "motor_damping": (25, 4),
           "projected_gravity": (29, 3)}
NOISE = {None: 0, "gaussian": 1, "uniform": 2}


def get_lib():
    global _LIB
    if _LIB is None:
        out = Path(tempfile.mkdtemp(prefix="wl_policy_obs_oracle_"))
        atexit.register(shutil.rmtree, out, True)
        fma = ["-mfma"] if " fma " in Path("/proc/cpuinfo").read_text().replace("\n", " ") else []
        cc = os.environ.get("WLO_CC", "/usr/bin/gcc")
        so = out / "libwl_policy_obs_oracle.so"
        subprocess.run([cc, "-O2", "-std=c11", *fma, "-fPIC", "-shared", "-ffp-contract=off", "-fno-fast-math", "-fopenmp",
                        "-o", str(so), str(HERE / "policy_obs_oracle.c"), "-lm"], check=True)
        lib = C.CDLL(str(so))
        vp = C.c_void_p
        lib.wlo_policy_observe.argtypes = [C.c_uint64, C.c_int32, C.c_int32, vp, C.c_int32, vp, vp, vp, vp, vp, vp, vp, vp, vp,
                                           C.c_int32, C.c_uint32, C.c_int32, vp]
        lib.wlo_policy_library.argtypes = [vp, C.c_int32, vp]
        lib.wlo_policy_obs_draw.argtypes = [C.c_uint64, C.c_uint32, C.c_uint32, C.c_int32, C.c_int32, C.c_int32]
        lib.wlo_policy_obs_draw.restype = C.c_float
        _LIB = lib
    return _LIB


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def columns(table) -> dict:
    """Per output column: src, noise kind, (na, nb) = (mean, std) or (n_min, n_max - n_min) with the span formed in double,
    clip flag and bounds, scale flag and value -- each parameter rounded to fp32."""
    cols = {k: [] for k in ("src", "noise", "na", "nb", "has_clip", "lo", "hi", "has_scale", "scale")}
    for name, noise, clip, scale in table:
        first, width = LIBRARY[name]
        sc = None if scale is None else ((float(scale),) if isinstance(scale, (int, float)) else tuple(float(s) for s in scale))
        for k in range(width):
            cols["src"].append(first + k)
            cols["noise"].append(NOISE[None if noise is None else noise[0]])
            a, b = (0.0, 0.0) if noise is None else (float(noise[1]), float(noise[2]))
            cols["na"].append(a)
            cols["nb"].append(b - a if noise is not None and noise[0] == "uniform" else b)
            cols["has_clip"].append(clip is not None)
            cols["lo"].append(0.0 if clip is None else float(clip[0]))
            cols["hi"].append(0.0 if clip is None else float(clip[1]))
            cols["has_scale"].append(sc is not None)
            cols["scale"].append(1.0 if sc is None else sc[0 if len(sc) == 1 else k])
    out = {}
    for k, v in cols.items():
        dt = np.uint8 if k in ("src", "noise", "has_clip", "has_scale") else np.float32
        out[k] = np.ascontiguousarray(np.asarray(v or [0], dtype=np.float64 if dt is np.float32 else np.int64).astype(dt))
    return out


def observe(seed, env_id_offset, st, table, corrupt, t, call_idx=-1) -> np.ndarray:
    """The policy row [N, Dp] of the state groups st [G, N, 4] for the step at t (call_idx -1) or an observe call."""
    st = np.ascontiguousarray(st, dtype=np.float32)
    n = st.shape[1]
    c = columns(table)
    dp = sum(LIBRARY[name][1] for name, *_ in table)
    out = np.zeros((n, max(dp, 1)), dtype=np.float32)
    get_lib().wlo_policy_observe(seed, env_id_offset, n, _p(st), dp, _p(c["src"]), _p(c["noise"]), _p(c["na"]), _p(c["nb"]),
                                 _p(c["has_clip"]), _p(c["lo"]), _p(c["hi"]), _p(c["has_scale"]), _p(c["scale"]), int(bool(corrupt)),
                                 t & 0xFFFFFFFF, call_idx, _p(out))
    return out[:, :dp]


def library(st) -> np.ndarray:
    """[N, 32] library floats of every env."""
    st = np.ascontiguousarray(st, dtype=np.float32)
    out = np.zeros((st.shape[1], 32), dtype=np.float32)
    get_lib().wlo_policy_library(_p(st), st.shape[1], _p(out))
    return out


def draw(seed, gid, t, call_idx, j, kind) -> np.float32:
    """The noise draw of column j: z (kind "gaussian") or u in [0, 1) (kind "uniform")."""
    return np.float32(get_lib().wlo_policy_obs_draw(seed, gid, t & 0xFFFFFFFF, call_idx, j, NOISE[kind]))
