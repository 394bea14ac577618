#!/usr/bin/env python
"""Record the reference's own env-cfg objects as data (tests/golden/ref_cfgs.json.gz + ref_cfgs_arrays.npz).

    python tests/golden/make_ref_cfgs.py <the reference's source/ directory>

The UNMODIFIED wheeledlab_tasks package is imported against the
stand-ins in shims/ (make_cfg_blobs.import_reference_tasks), which registers the four gym ids; every registered train and
play cfg is instantiated (num_envs = 4096) and written out field by field: values as they are, the functions a term refers
to and the classes a field names by name only, large boolean / numeric tables (the Visual traversability map) into the npz.
tests/recorded_cfgs.py rebuilds objects with the same attribute names, values, field order and type / function names, which is
everything wheeledlab_b200.compat reads, so tests/test_compat_cpu.py lowers the reference cfgs without the reference tree.
"""
import gzip
import importlib.util
import json
import sys
import types
from pathlib import Path

import numpy as np

HERE = Path(__file__).resolve().parent
OUT_JSON, OUT_NPZ = HERE / "ref_cfgs.json.gz", HERE / "ref_cfgs_arrays.npz"


def _is_table(v):
    return isinstance(v, (list, tuple)) and len(v) > 64 and all(isinstance(x, (list, tuple)) for x in v[:4])


class _Recorder:
    def __init__(self):
        self.arrays = {}

    def rec(self, v, path):
        if v is None or isinstance(v, (bool, int, str)):
            return v
        if isinstance(v, float):
            return v if np.isfinite(v) else {"__float__": repr(v)}
        if isinstance(v, np.ndarray) or _is_table(v):
            key = f"a{len(self.arrays)}"
            self.arrays[key] = np.asarray(v)
            return {"__array__": key, "path": path}
        if isinstance(v, (types.FunctionType, types.BuiltinFunctionType, types.MethodType)):
            return {"__func__": v.__name__}
        if isinstance(v, type):
            return {"__class__": v.__name__}
        if isinstance(v, (list, tuple)):
            return {"__tuple__" if isinstance(v, tuple) else "__list__": [self.rec(x, f"{path}[{i}]") for i, x in enumerate(v)]}
        if isinstance(v, dict):
            return {"__dict__": [[k, self.rec(x, f"{path}.{k}")] for k, x in v.items()]}
        names = getattr(v, "_cfg_fields", None)
        if names is not None:
            return {"__cfg__": type(v).__name__, "fields": [[k, self.rec(getattr(v, k), f"{path}.{k}")] for k in names]}
        if hasattr(v, "__dict__") and not isinstance(v, types.ModuleType):
            return {"__obj__": type(v).__name__, "fields": [[k, self.rec(x, f"{path}.{k}")] for k, x in vars(v).items()]}
        if callable(v) and hasattr(v, "__name__"):
            return {"__func__": v.__name__}
        return {"__repr__": repr(v)}


def main():
    spec = importlib.util.spec_from_file_location("make_cfg_blobs", HERE / "make_cfg_blobs.py")
    mk = importlib.util.module_from_spec(spec); spec.loader.exec_module(mk)
    gym = mk.import_reference_tasks(Path(sys.argv[1]))
    r = _Recorder()
    registry = {}
    for gid in gym.registry:
        s = gym.spec(gid)
        ent = {"entry_point": s.entry_point, "kwargs": {}, "cfgs": {}}
        for key, val in s.kwargs.items():
            if isinstance(val, type):
                cfg = val()
                cfg.scene.num_envs = 4096
                ent["kwargs"][key] = {"__class__": val.__name__}
                ent["cfgs"][key] = r.rec(cfg, f"{gid}.{key}")
            else:
                ent["kwargs"][key] = val
        registry[gid] = ent
    text = json.dumps({"num_envs": 4096, "registry": registry}, indent=None, separators=(",", ":")) + "\n"
    OUT_JSON.write_bytes(gzip.compress(text.encode(), mtime=0))
    np.savez_compressed(OUT_NPZ, **r.arrays)
    print(OUT_JSON, OUT_JSON.stat().st_size, "bytes;", OUT_NPZ, OUT_NPZ.stat().st_size, "bytes")


if __name__ == "__main__":
    main()
