"""The reference's env-cfg objects, rebuilt from the record in tests/golden/ref_cfgs.json.gz (tests/golden/make_ref_cfgs.py).

Every object has the recorded attributes in the recorded order (``_cfg_fields`` for config classes), a type of the recorded
name, and stand-in functions / classes that carry the recorded ``__name__``: what wheeledlab_b200.compat reads to lower a cfg.
A recorded function cannot be called (the reference's code is not part of this repository)."""
from __future__ import annotations

import gzip
import json
from pathlib import Path

import numpy as np

GOLDEN = Path(__file__).resolve().parent / "golden"
_types: dict = {}


class RecordedCfg:
    def __repr__(self):
        return f"{type(self).__name__}(" + ", ".join(f"{k}={v!r}" for k, v in vars(self).items() if not k.startswith("_")) + ")"


def _type(name, base):
    key = (name, base)
    if key not in _types:
        _types[key] = type(name, (base,), {})
    return _types[key]


def _func(name):
    def recorded(*args, **kwargs):
        raise NotImplementedError(f"{name}: a recorded reference function (not callable)")
    recorded.__name__ = recorded.__qualname__ = name
    return recorded


class _Builder:
    def __init__(self, arrays):
        self.arrays = arrays
        self.funcs: dict = {}

    def build(self, v):
        if not isinstance(v, dict):
            return v
        if "__float__" in v:
            return float(v["__float__"])
        if "__array__" in v:
            return self.arrays[v["__array__"]].copy()
        if "__func__" in v:
            return self.funcs.setdefault(v["__func__"], _func(v["__func__"]))
        if "__class__" in v:
            return _type(v["__class__"], object)
        if "__tuple__" in v:
            return tuple(self.build(x) for x in v["__tuple__"])
        if "__list__" in v:
            return [self.build(x) for x in v["__list__"]]
        if "__dict__" in v:
            return {k: self.build(x) for k, x in v["__dict__"]}
        if "__repr__" in v:
            return slice(None) if v["__repr__"] == "slice(None, None, None)" else v["__repr__"]
        obj = _type(v.get("__cfg__") or v["__obj__"], RecordedCfg)()
        for k, x in v["fields"]:
            setattr(obj, k, self.build(x))
        if "__cfg__" in v:
            obj._cfg_fields = [k for k, _ in v["fields"]]
        return obj


def load():
    """{gym id: {"entry_point": str, "kwargs": {key: str | recorded class}, "cfgs": {key: factory of a fresh cfg object}}}"""
    rec = json.loads(gzip.decompress((GOLDEN / "ref_cfgs.json.gz").read_bytes()))
    with np.load(GOLDEN / "ref_cfgs_arrays.npz") as z:
        arrays = {k: z[k] for k in z.files}
    out = {}
    for gid, ent in rec["registry"].items():
        b = _Builder(arrays)
        out[gid] = {"entry_point": ent["entry_point"], "kwargs": {k: b.build(v) for k, v in ent["kwargs"].items()},
                    "cfgs": {k: (lambda _v=v: _Builder(arrays).build(_v)) for k, v in ent["cfgs"].items()}}
    return out
