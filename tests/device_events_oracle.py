"""The device event terms' CPU twin (tests/device_events_oracle.c): TEST INFRASTRUCTURE ONLY.

The C file is compiled, with the oracle's own flags, into a temporary directory on first use (the source tree may be
read-only).  A table is a list of (mode, interval_range_s or None, six (lo, hi) velocity ranges), as
``WheeledSim.set_device_events`` takes it.  ``init`` draws the interval terms' timers; ``step`` runs one step in place on
time_left [n_interval_terms, N] f32 and vel [N, 6] f32 (x, y, z, roll, pitch, yaw)."""
from __future__ import annotations

import atexit
import ctypes as C
import os
import shutil
import subprocess
import tempfile
from pathlib import Path

import numpy as np

import event_timers_oracle as eo

HERE = Path(__file__).resolve().parent
_LIB = None


def get_lib():
    global _LIB
    if _LIB is None:
        out = Path(tempfile.mkdtemp(prefix="wl_device_events_oracle_"))
        atexit.register(shutil.rmtree, out, True)
        fma = ["-mfma"] if " fma " in Path("/proc/cpuinfo").read_text().replace("\n", " ") else []
        cc = os.environ.get("WLO_CC", "/usr/bin/gcc")
        so = out / "libwl_device_events_oracle.so"
        subprocess.run([cc, "-O2", "-std=c11", *fma, "-fPIC", "-shared", "-ffp-contract=off", "-fno-fast-math", "-fopenmp",
                        "-o", str(so), str(HERE / "device_events_oracle.c"), "-lm"], check=True)
        lib = C.CDLL(str(so))
        vp = C.c_void_p
        lib.wlo_device_events.argtypes = [C.c_uint64, C.c_int32, C.c_int32, C.c_int32, vp, vp, vp, C.c_int32, vp, C.c_float, vp, vp, vp,
                                          C.c_int64]
        _LIB = lib
    return _LIB


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _timer_ranges(table):
    return [tuple(r) for mode, r, _ in table if mode == "interval"]


def init(seed, env_id_offset, n, table) -> np.ndarray:
    """The interval terms' timers as wl_set_device_events draws them: [n_interval_terms, N] f32."""
    ranges = _timer_ranges(table)
    return eo.init(seed, env_id_offset, n, ranges) if ranges else np.zeros((0, n), np.float32)


def step(seed, env_id_offset, table, step_dt, done, time_left, vel, step_counter):
    """One step of every term, in place on time_left and vel [N, 6]."""
    n = vel.shape[0]
    slot, j = [], 0
    for mode, _, _ in table:
        slot.append(j if mode == "interval" else -1)
        j += mode == "interval"
    slot = np.asarray(slot or [0], dtype=np.int32)
    lo = np.ascontiguousarray([[r[0] for r in rr] for _, _, rr in table] or [[0.0] * 6], dtype=np.float32)
    hi = np.ascontiguousarray([[r[1] for r in rr] for _, _, rr in table] or [[0.0] * 6], dtype=np.float32)
    tlh = np.ascontiguousarray(_timer_ranges(table) or [(0.0, 0.0)], dtype=np.float32).reshape(-1)
    done = np.ascontiguousarray(done, dtype=np.uint8)
    assert vel.dtype == np.float32 and vel.flags.c_contiguous and time_left.dtype == np.float32 and time_left.flags.c_contiguous
    get_lib().wlo_device_events(seed, env_id_offset, n, len(table), _p(slot), _p(lo), _p(hi), j, _p(tlh), np.float32(step_dt), _p(done),
                                _p(time_left), _p(vel), step_counter)
