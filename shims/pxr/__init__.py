"""Stand-in for `pxr` (OpenUSD) as far as the UNMODIFIED reference touches it at import time:
wheeledlab_tasks/visual/utils/__init__.py:154-186 (create_geometry) builds a Usd.Stage with the 2-colour plane mesh and saves it
for the RTX scene.  The fused-step env renders that plane from the traversability map itself (wl_camera_kernel), so the stage
calls are absorbed: every attribute access / call returns an inert object and nothing is written to disk."""


class _Absorb:
    def __getattr__(self, name):
        if name.startswith("__") and name.endswith("__"):
            raise AttributeError(name)
        return _Absorb()

    def __call__(self, *a, **k):
        return _Absorb()

    def __bool__(self):
        return True

    def __iter__(self):
        return iter(())


class _Gf(_Absorb):
    @staticmethod
    def Vec3f(*a):
        return tuple(float(x) for x in (a[0] if len(a) == 1 and hasattr(a[0], "__len__") else a))

    Vec3d = Vec3f


Usd, UsdGeom, UsdPhysics, UsdShade, Sdf, Vt = _Absorb(), _Absorb(), _Absorb(), _Absorb(), _Absorb(), _Absorb()
Gf = _Gf()
