"""The integrator sub-step loop of the Drift-family duo kernel, read from the compiled SASS (tools/substep_sass.py).

The report finds the loop in every duo instantiation.  The two shipped step specs run every pass without a divergent
region (dc_limits_sel and the selected tyre direction, DESIGN.md 6e), and their pass stays at most as long as this
build's: a pass is one env warp's dependent instruction stream.  (ptxas still guards the butterfly with a BRA.DIV.)"""
import importlib.util
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent
SPEC_KEYS = (0x80010475, 0x80010476)          # SPEC_DRIFT_RWD (Drift) and SPEC_DRIFT_4WD (HOUND-4WD)
MAX_INSTRUCTIONS_PER_PASS = 349

_spec = importlib.util.spec_from_file_location("substep_sass", ROOT / "tools" / "substep_sass.py")
sass = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(sass)
pytestmark = pytest.mark.skipif(sass.tools() is None, reason="needs nvcc and cuobjdump")


@pytest.fixture(scope="module")
def rows(tmp_path_factory):
    cubin = sass.compile_cubin(ROOT, tmp_path_factory.mktemp("sass") / "wl_api.cubin")
    return {(r["fan"], r["spec"]): r for r in sass.report(cubin)}


def test_every_duo_instantiation_has_a_substep_loop(rows):
    assert {(0, 0), (1, 0), (2, 0), *((0, k) for k in SPEC_KEYS)} <= set(rows)
    for key, r in rows.items():
        assert "error" not in r, (key, r)
        assert r["mix"].get("SHFL", 0) == 12, (key, r["mix"])           # the force / torque butterfly, 6 values x 2 steps
        assert 0 < r["chain_two_passes"], (key, r)


@pytest.mark.parametrize("key", SPEC_KEYS)
def test_spec_pass_is_branch_free(rows, key):
    r = rows[(0, key)]
    assert r["bssy"] == 0 and r["bsync"] == 0 and r["bra"] == 1, r      # only the loop's back edge
    assert r["instructions_per_pass"] <= MAX_INSTRUCTIONS_PER_PASS, r
