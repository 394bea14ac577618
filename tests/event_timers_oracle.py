"""The interval timers' CPU twin (tests/event_timers_oracle.c): TEST INFRASTRUCTURE ONLY.

The C file is compiled, with the oracle's own flags, into a temporary directory on first use (the source tree may be
read-only).  ``init`` and ``step`` take and return numpy arrays: time_left [n_terms, N] f32, fired [n_terms, N] u8."""
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


def get_lib():
    global _LIB
    if _LIB is None:
        out = Path(tempfile.mkdtemp(prefix="wl_event_timers_oracle_"))
        atexit.register(shutil.rmtree, out, True)
        fma = ["-mfma"] if " fma " in Path("/proc/cpuinfo").read_text().replace("\n", " ") else []
        cc = os.environ.get("WLO_CC", "/usr/bin/gcc")
        so = out / "libwl_event_timers_oracle.so"
        subprocess.run([cc, "-O2", "-std=c11", *fma, "-fPIC", "-shared", "-ffp-contract=off", "-fno-fast-math", "-fopenmp",
                        "-o", str(so), str(HERE / "event_timers_oracle.c"), "-lm"], check=True)
        lib = C.CDLL(str(so))
        vp = C.c_void_p
        lib.wlo_event_timers_init.argtypes = [C.c_uint64, C.c_int32, C.c_int32, C.c_int32, vp, vp]
        lib.wlo_event_timers.argtypes = [C.c_uint64, C.c_int32, C.c_int32, C.c_int32, vp, C.c_float, vp, vp, vp, C.c_int64]
        _LIB = lib
    return _LIB


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def init(seed, env_id_offset, n, ranges) -> np.ndarray:
    lo_hi = np.ascontiguousarray(ranges, dtype=np.float32).reshape(-1)
    tl = np.zeros((len(ranges), n), dtype=np.float32)
    get_lib().wlo_event_timers_init(seed, env_id_offset, n, len(ranges), _p(lo_hi), _p(tl))
    return tl


def step(seed, env_id_offset, ranges, step_dt, done, time_left, step_counter):
    """One step in place on time_left; returns fired."""
    lo_hi = np.ascontiguousarray(ranges, dtype=np.float32).reshape(-1)
    n = time_left.shape[1]
    done = np.ascontiguousarray(done, dtype=np.uint8)
    fired = np.zeros(time_left.shape, dtype=np.uint8)
    get_lib().wlo_event_timers(seed, env_id_offset, n, len(ranges), _p(lo_hi), np.float32(step_dt), _p(done), _p(time_left),
                               _p(fired), step_counter)
    return fired
