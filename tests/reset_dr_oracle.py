"""The oracle with the reset-mode DR events (tests/reset_dr_oracle.c): TEST INFRASTRUCTURE ONLY.

The C twin is compiled, with the oracle's own flags, into a temporary directory on first use (the source tree may be
read-only); ``Oracle(cfg, heightfield, mask)`` is ``oracle_lib.Oracle`` on that library with the handle's mask set."""
from __future__ import annotations

import atexit
import ctypes as C
import os
import shutil
import subprocess
import tempfile
from pathlib import Path

import oracle_lib

HERE = Path(__file__).resolve().parent
_LIB = None


def get_lib():
    global _LIB
    if _LIB is None:
        out = Path(tempfile.mkdtemp(prefix="wl_reset_dr_oracle_"))
        atexit.register(shutil.rmtree, out, True)
        fma = ["-mfma"] if " fma " in Path("/proc/cpuinfo").read_text().replace("\n", " ") else []
        cc = os.environ.get("WLO_CC", "/usr/bin/gcc")
        so = out / "libwl_reset_dr_oracle.so"
        subprocess.run([cc, "-O2", "-std=c11", *fma, "-fPIC", "-shared", "-ffp-contract=off", "-fno-fast-math", "-fopenmp",
                        "-o", str(so), str(HERE / "reset_dr_oracle.c"), "-lm"], check=True)
        _LIB = oracle_lib._load(so)
        _LIB.wlo_set_reset_events.argtypes = [C.c_void_p, C.c_uint32]
    return _LIB


class Oracle(oracle_lib.Oracle):
    """oracle_lib.Oracle whose step, step_terms and reset apply the reset-mode DR events of `mask` (WL_RESET_EV_* bits)."""

    def __init__(self, cfg, heightfield=None, mask=0, threads=1):
        self._lib = get_lib()
        super().__init__(cfg, heightfield, threads=threads)
        assert self.set_reset_events(mask) == 0

    def set_reset_events(self, mask) -> int:
        """wlo_set_reset_events: 0, or WL_EINVAL with the mask left as it was."""
        return self.lib.wlo_set_reset_events(self._h, mask)

    @property
    def lib(self):
        return self._lib

    @lib.setter
    def lib(self, _):
        pass                                      # (oracle_lib.Oracle.__init__ assigns the plain oracle; this one is kept)
