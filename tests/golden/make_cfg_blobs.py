#!/usr/bin/env python
"""Write the lowered wl_config of every registered task as a binary blob (tests/golden/cfg_blobs/<name>.bin).

Two producers must agree byte for byte (tests/test_compat_cpu.py, tests/test_gpu_parity.py):
  * the package's own restatement of the reference configuration (wheeledlab_b200.tasks.make_task), and
  * the lowering of the REFERENCE'S OWN cfg objects (wheeledlab_b200.compat.spec_from_reference_cfg), imported from
    the reference's source/ directory when its path is given as the first argument (recorded as <name>.ref.bin).
The blobs also let non-Python hosts (examples/c_host) and bench.py's reference arm build a task without importing the package.
num_envs = 4096, seed = 42, env_id_offset = 0 in every blob (the first fields of wl_config; consumers patch them).
"""
import ctypes as C
import sys
from pathlib import Path

HERE = Path(__file__).resolve().parent
ROOT = HERE.parent.parent
sys.path.insert(0, str(ROOT))
OUT = HERE / "cfg_blobs"

TASKS = {"drift": "Isaac-MushrDriftRL-v0", "f1tenth_drift": "Isaac-F1TenthDriftRL-v0", "elevation": "Isaac-MushrElevationRL-v0",
         "visual": "Isaac-MushrVisualRL-v0", "hound_4wd": "hound_4wd"}


def blob(cfg) -> bytes:
    return C.string_at(C.addressof(cfg), C.sizeof(cfg))


def import_reference_tasks(ref: Path):
    """Import the UNMODIFIED wheeledlab_tasks package of the reference's source/ directory `ref` against the stand-ins in shims/ (gymnasium, isaaclab,
    pxr, matplotlib).  Importing it registers the four gym ids (wheeledlab_tasks/__init__.py:14-63) and -- quirk Q10 -- builds the
    Visual traversability map and tries to create <assets>/data/rgb_maps: the reference tree is read-only here, so that one
    makedirs is skipped."""
    import os
    ref = Path(ref)
    sys.path[:0] = [str(ROOT / "shims"), str(ref / "wheeledlab"), str(ref / "wheeledlab_assets"), str(ref / "wheeledlab_tasks")]
    real = os.makedirs

    def makedirs(path, *a, **k):
        if str(path).startswith(str(ref)):
            return None
        return real(path, *a, **k)

    top = sys.modules.get("wheeledlab_tasks")
    if top is not None and getattr(top, "__file__", None) is None:       # a path-only stub of another test (skips __init__): drop it
        for k in [k for k in sys.modules if k == "wheeledlab_tasks" or k.startswith("wheeledlab_tasks.")]:
            del sys.modules[k]
    os.makedirs = makedirs
    try:
        import wheeledlab_tasks  # noqa: F401
    finally:
        os.makedirs = real
    import gymnasium as gym
    return gym


def main():
    import numpy as np
    import wheeledlab_b200 as wl
    OUT.mkdir(exist_ok=True)
    for name, tid in TASKS.items():
        spec = wl.make_task(tid, num_envs=4096, seed=42)
        (OUT / f"{name}.bin").write_bytes(blob(spec.cfg))
        print(name, C.sizeof(spec.cfg), "bytes")
    if len(sys.argv) > 1:                                # the reference's source/ directory: lower its own cfg objects
        from wheeledlab_b200.compat import spec_from_reference_cfg
        gym = import_reference_tasks(Path(sys.argv[1]))
        for gid in gym.registry:
            for key, suffix in (("env_cfg_entry_point", "ref"), ("play_env_cfg_entry_point", "play.ref")):
                cls = gym.spec(gid).kwargs.get(key)
                if cls is None:
                    continue
                cfg = cls()
                cfg.scene.num_envs = 4096
                got = spec_from_reference_cfg(cfg)
                (OUT / f"{gid}.{suffix}.bin").write_bytes(blob(got.cfg))
                if "Visual" in gid and suffix == "ref":
                    np.savez_compressed(OUT / "visual_ref_map.npz", map=np.asarray(cfg.scene.terrain.traversability_hashmap, dtype=bool))
                print(gid, suffix)


if __name__ == "__main__":
    main()
