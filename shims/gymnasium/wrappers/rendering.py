"""gymnasium.wrappers.rendering stand-in (wheeledlab_rl/utils/custom_record_video.py imports RecordVideo from here)."""
from ..core import Wrapper


class RecordVideo(Wrapper):
    def __init__(self, env, *a, **k):
        raise NotImplementedError("video recording needs the reference's RTX viewport (out of scope for the fused-step env: render() is None)")
