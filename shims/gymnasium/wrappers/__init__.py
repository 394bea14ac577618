"""gymnasium.wrappers stand-in: RecordVideo needs the Omniverse viewport the reference renders through (out of scope)."""
from ..core import Wrapper
from . import rendering  # noqa: F401


class RecordVideo(Wrapper):
    def __init__(self, env, *a, **k):
        raise NotImplementedError("video recording needs the reference's RTX viewport (out of scope for the fused-step env: render() is None)")
