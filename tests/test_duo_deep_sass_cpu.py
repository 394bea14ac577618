"""The deep-chained duo kernel (wl_step_duo_deep_kernel: four env warps and one aux warp per CTA, DESIGN.md 6e), read from the
compiled SASS (tools/substep_sass.py, tools/phase_sass.py, cuobjdump -res-usage).

Four CTAs of 160 threads fit on an SM at up to 96 registers a thread (5 warps a scheduler), so every instantiation stays
there without a spill.  The env warps run the shallow kernel's code: the shipped specs' sub-step pass is branch-free and
their tail select-shaped.  The aux warp serves 32 envs, one per lane; its reward tail stays select-shaped, with the episode
log's REDs issued by lanes 0..15 under a predicate."""
import importlib.util
import re
import subprocess
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent
SPEC_KEYS = (0x80010475, 0x80010476)          # SPEC_DRIFT_RWD (Drift) and SPEC_DRIFT_4WD (HOUND-4WD)
MAX_REGISTERS = 96
MAX_INSTRUCTIONS_PER_PASS = 352
ENV_TAIL = {"instructions": 320, "bssy": 3, "call": 1}
AUX_TAIL = {"instructions": 480, "bssy": 3, "call": 1}


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
def cubin(tmp_path_factory):
    return ss.compile_cubin(ROOT, tmp_path_factory.mktemp("sass") / "wl_api.cubin")


@pytest.fixture(scope="module")
def phases(cubin):
    return {r["spec"]: r for r in ps.report(cubin) if r["fan"] == ss.DEEP}


@pytest.fixture(scope="module")
def loops(cubin):
    return {r["spec"]: r for r in ss.report(cubin) if r["fan"] == ss.DEEP}


@pytest.fixture(scope="module")
def resources(cubin):
    """{K: {"REG": .., "STACK": .., "LOCAL": ..}} of every wl_step_duo_deep_kernel<K>"""
    txt = subprocess.run([ss.tools()[1], "-res-usage", str(cubin)], check=True, capture_output=True, text=True).stdout
    out = {}
    for m in re.finditer(r"Function _Z23wl_step_duo_deep_kernelILj(\d+)E\S*:\s*\n\s*(.*)", txt):
        out[int(m.group(1))] = {k: int(v) for k, v in re.findall(r"(REG|STACK|LOCAL):(\d+)", m.group(2))}
    return out


def test_every_deep_instantiation_is_reported(phases, loops, resources):
    assert {0, *SPEC_KEYS} <= set(phases) and set(phases) == set(loops) == set(resources), (set(phases), set(resources))
    for k, r in loops.items():
        assert "error" not in r and r["mix"].get("SHFL", 0) == 12, (hex(k), r)


def test_deep_kernels_fit_four_ctas_per_sm_without_spills(resources):
    for k, r in resources.items():
        assert r["REG"] <= MAX_REGISTERS and r["STACK"] == 0 and r["LOCAL"] == 0, (hex(k), r)


@pytest.mark.parametrize("key", SPEC_KEYS)
def test_deep_spec_pass_is_branch_free(loops, key):
    r = loops[key]
    assert r["bssy"] == 0 and r["bsync"] == 0 and r["bra"] == 1, r
    assert r["instructions_per_pass"] <= MAX_INSTRUCTIONS_PER_PASS, r


@pytest.mark.parametrize("key", SPEC_KEYS)
def test_deep_tails_are_select_shaped(phases, key):
    env, aux = phases[key]["env: bar.arrive 2 -> exit"], phases[key]["aux: bar.sync 2 -> exit"]
    assert env["instructions"] <= ENV_TAIL["instructions"] and env["bssy"] <= ENV_TAIL["bssy"] and env["call"] <= ENV_TAIL["call"], env
    assert aux["instructions"] <= AUX_TAIL["instructions"] and aux["bssy"] <= AUX_TAIL["bssy"] and aux["call"] <= AUX_TAIL["call"], aux
