"""The Drift-family duo kernel's segments outside the sub-step loop, read from the compiled SASS (tools/phase_sass.py).

For the two shipped step specs the env warp's tail (bar.arrive 2 to exit) runs the euler angles, the reset / push choice, the
observation slice and the state stores as selects (DESIGN.md 6e).  What divergent regions are left there: the atan2
quotient's IEEE division (its slow path serves subnormal quotients) and the warp-uniform choice between the staged and the
element-wise observation stores.  The aux warp's reward tail (bar.sync 2 to exit) likewise: its roots without slow-path
calls, the weighing and the stores by select and predicate, the episode log reduced over the eight env lanes; left there:
the slip angle's IEEE division and the lanes-0..7 region.  The aux warp loads the reward weights only after bar.arrive 1."""
import importlib.util
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent
SPEC_KEYS = (0x80010475, 0x80010476)          # SPEC_DRIFT_RWD (Drift) and SPEC_DRIFT_4WD (HOUND-4WD)
ENV_TAIL = {"instructions": 320, "bssy": 3, "call": 1}
AUX_TAIL = {"instructions": 420, "bssy": 3, "call": 1}


def _load(name):
    spec = importlib.util.spec_from_file_location(name, ROOT / "tools" / f"{name}.py")
    mod = importlib.util.module_from_spec(spec)
    sys.modules[name] = mod
    spec.loader.exec_module(mod)
    return mod


sys.path.insert(0, str(ROOT / "tools"))
ss = _load("substep_sass")
ps = _load("phase_sass")
pytestmark = pytest.mark.skipif(ss.tools() is None, reason="needs nvcc and cuobjdump")


@pytest.fixture(scope="module")
def rows(tmp_path_factory):
    cubin = ss.compile_cubin(ROOT, tmp_path_factory.mktemp("sass") / "wl_api.cubin")
    return {(r["fan"], r["spec"]): r for r in ps.report(cubin)}


@pytest.mark.parametrize("key", SPEC_KEYS)
def test_env_tail_is_select_shaped(rows, key):
    s = rows[(0, key)]["env: bar.arrive 2 -> exit"]
    assert s["instructions"] <= ENV_TAIL["instructions"], s
    assert s["bssy"] <= ENV_TAIL["bssy"] and s["call"] <= ENV_TAIL["call"], s


@pytest.mark.parametrize("key", SPEC_KEYS)
def test_aux_reward_tail_is_select_shaped(rows, key):
    s = rows[(0, key)]["aux: bar.sync 2 -> exit"]
    assert s["instructions"] <= AUX_TAIL["instructions"], s
    assert s["bssy"] <= AUX_TAIL["bssy"] and s["call"] <= AUX_TAIL["call"], s


@pytest.mark.parametrize("key", SPEC_KEYS)
def test_env_prologue_has_no_slow_path_call(rows, key):
    assert rows[(0, key)]["env: entry -> bar.sync 1"]["call"] == 0, rows[(0, key)]


def test_generic_duo_tail_keeps_its_branches(rows):
    # the generic body (K = 0) is not specialised: the branches it had are still there
    assert rows[(0, 0)]["env: bar.arrive 2 -> exit"]["bssy"] > ENV_TAIL["bssy"], rows[(0, 0)]
