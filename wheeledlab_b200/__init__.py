"""wheeledlab_b200 -- H100-native fused step for the WheeledLab Drift / Elevation / Visual tasks.

Importing the package loads ``libwheeledlab_b200.so`` (hand-written sm_90a kernels behind a C ABI);
it raises if the library has not been built -- there is no CPU or eager-PyTorch fallback.
"""
from ._lib import LIB_PATH, WlConfig, WlError, lib  # noqa: F401
from .tasks import GYM_IDS, TaskSpec, drift_task, elevation_task, make_task, visual_task  # noqa: F401
from .sim import WheeledSim, upload_graph  # noqa: F401
from .env import ManagerBasedRLEnv, make  # noqa: F401

__version__ = "0.1.0"
