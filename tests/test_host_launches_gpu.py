"""The kernel launches of one call of every entry that steps the envs or writes the built-in row: the wl_launch_count
increment of each call, on every task (Visual with and without the camera), with and without row terms and reset-mode DR
events, with device terms and device events in wl_step_terms, on consecutive and jumping counters, a device counter, and a
host counter that lands on a curriculum boundary.  The bit-parity suites do not see a launch that was dropped, repeated or
moved between entries without changing the outputs; these counts do."""
import pytest
import torch

pytestmark = pytest.mark.gpu

if not torch.cuda.is_available():
    pytest.skip("needs a CUDA device", allow_module_level=True)

import wheeledlab_b200 as wl                                   # noqa: E402
from wheeledlab_b200 import policy as P                        # noqa: E402
from wheeledlab_b200._lib import WL_ROW_TASK_TERMS, WlError    # noqa: E402
from wheeledlab_b200.distributed import RolloutSlab            # noqa: E402
from wheeledlab_b200.sim import WheeledSim                     # noqa: E402

DEV = "cuda:0"
N = 64
# In call order; "L" is the config's max_episode_length, the curriculum's boundary (the Visual task has no curriculum).
CALLS = ["reset", "step 0", "step 5 (jump)", "stage_a 6", "stage_b 6", "stage_a 20 (jump)", "stage_b1 20", "stage_b2 20",
         "step_terms 21 (no device terms: wl_step)", "observe", "act_step 22", "act_infer_step 23", "rollout 24..25",
         "step L-1 (boundary)", "rollout 2L-2..2L-1 (boundary)", "step device counter + 0", "step_terms 1, device terms",
         "step_terms 2, device terms + log", "step_terms 3, device terms + log + events", "step_terms 4, device events",
         "step_terms L-1, device events (boundary)", "step with device events"]
R = None        # refused (WlError) before any launch
# (task, row terms, reset events) -> the increment of each call above
EXPECTED = {
    ("drift", False, False):         (1, 1, 3, 1, 1, 3, 1, 1, 1, 1, 1, 1, 1, 4, 4, 3, 3, 4, 6, 4, 7, R),
    ("drift", False, True):          (2, 2, 4, 1, 2, 3, 2, 1, 2, 1, 2, 2, R, 5, R, 4, 4, 5, 7, 5, 8, R),
    ("elevation", False, False):     (1, 2, 4, 1, 2, 3, 1, 2, 2, 2, R, R, R, 5, R, 4, 4, 5, 7, 5, 8, R),
    ("elevation", False, True):      (2, 3, 5, 1, 3, 3, 2, 2, 3, 2, R, R, R, 6, R, 5, 5, 6, 8, 6, 9, R),
    ("elevation", True, False):      (1, 2, 4, 1, 2, 3, 1, 2, 2, 2, R, R, R, 5, R, 4, 4, 5, 7, 5, 8, R),
    ("elevation", True, True):       (2, 3, 5, 1, 3, 3, 2, 2, 3, 2, R, R, R, 6, R, 5, 5, 6, 8, 6, 9, R),
    ("visual", False, False):        (1, 1, 3, 1, 1, 3, 1, 1, 1, 1, 1, 1, 1, 3, 3, 3, 3, 4, 6, 4, 6, R),
    ("visual", False, True):         (2, 2, 4, 1, 2, 3, 2, 1, 2, 1, 2, 2, R, 4, R, 4, 4, 5, 7, 5, 7, R),
    ("visual", True, False):         (1, 2, 4, 1, 2, 3, 1, 2, 2, 2, R, R, R, 4, R, 4, 4, 5, 7, 5, 7, R),
    ("visual", True, True):          (2, 3, 5, 1, 3, 3, 2, 2, 3, 2, R, R, R, 5, R, 5, 5, 6, 8, 6, 8, R),
    ("visual+camera", False, False): (1, 2, 4, 1, 2, 3, 1, 2, 2, 2, R, R, R, 4, R, 4, 4, 5, 7, 5, 7, R),
    ("visual+camera", False, True):  (2, 3, 5, 1, 3, 3, 2, 2, 3, 2, R, R, R, 5, R, 5, 5, 6, 8, 6, 8, R),
    ("visual+camera", True, False):  (1, 3, 5, 1, 3, 3, 1, 3, 3, 3, R, R, R, 5, R, 5, 5, 6, 8, 6, 8, R),
    ("visual+camera", True, True):   (2, 4, 6, 1, 4, 3, 2, 3, 4, 3, R, R, R, 6, R, 6, 6, 7, 9, 7, 9, R),
}


def _spec(task):
    if task == "drift":
        return wl.drift_task(num_envs=N, seed=5)
    if task == "elevation":
        return wl.elevation_task(num_envs=N, seed=5)
    return wl.visual_task(num_envs=N, seed=5, camera="aug" if task == "visual+camera" else None, randomize=True)


def _launches(task, rows, events):
    spec = _spec(task)
    sim = WheeledSim(spec, DEV)
    if rows:
        sim.set_row_terms(WL_ROW_TASK_TERMS[task.split("+")[0]])
    if events:
        sim.set_reset_events(material=True)
    sim.startup()
    L = int(spec.cfg.max_episode_length)
    D = sim.obs_dim
    act = torch.zeros((N, 2), dtype=torch.float32, device=DEV)
    out = (torch.empty((N, D), dtype=torch.float32, device=DEV), torch.empty(N, dtype=torch.float32, device=DEV),
           torch.empty(N, dtype=torch.uint8, device=DEV), torch.empty(N, dtype=torch.uint8, device=DEV))
    _, blob_floats = P.blob_layout(D)
    blob = torch.zeros(blob_floats, dtype=torch.float32, device=DEV)
    actions, mean = torch.zeros((N, 2), dtype=torch.float32, device=DEV), torch.zeros((N, 2), dtype=torch.float32, device=DEV)
    lp, val = torch.zeros(N, dtype=torch.float32, device=DEV), torch.zeros(N, dtype=torch.float32, device=DEV)
    slab = RolloutSlab(2, N, D, 2, DEV)
    logs = torch.zeros((2, 16), dtype=torch.float32, device=DEV)
    term_log = torch.zeros(8, dtype=torch.float32, device=DEV)
    bits = torch.zeros(N, dtype=torch.uint8, device=DEV)

    def stage_a(t):
        bits.copy_(sim.step_stage_a(act, t)[1])

    push = [("interval", (0.1, 0.2), [(-0.5, 0.5)] * 6)]
    calls = [
        lambda: sim.reset(None, 0),
        lambda: sim.step(act, 0, out=out),
        lambda: sim.step(act, 5, out=out),
        lambda: stage_a(6),
        lambda: sim.step_stage_b(bits, 6),
        lambda: stage_a(20),
        lambda: sim.step_stage_b1(bits, 20),
        lambda: sim.step_stage_b2(20),
        lambda: sim.step_terms(act, 21, out=out),
        lambda: sim.observe(21, 0),
        lambda: P.act_step(sim, out[0], blob, actions, mean, lp, val, out, None, 22),
        lambda: P.act_infer_step(sim, out[0], blob, actions, out, None, 23),
        lambda: sim.rollout(2, 24, slab, logs),
        lambda: sim.step(act, L - 1, out=out),
        lambda: sim.rollout(2, 2 * L - 2, slab, logs),
        lambda: sim.step(act, WheeledSim.device_counter_plus(0), out=out),
        lambda: sim.step_terms(act, 1, out=out),
        lambda: sim.step_terms(act, 2, out=out, term_log=term_log),
        lambda: sim.step_terms(act, 3, out=out, term_log=term_log),
        lambda: sim.step_terms(act, 4, out=out),
        lambda: sim.step_terms(act, L - 1, out=out),
        lambda: sim.step(act, L, out=out),
    ]
    # set-up before a call (its own launches are not counted): device terms from the 17th call on, device events from the
    # 19th, and no device terms from the 20th
    setup = {16: lambda: sim.set_device_terms([(1, 0, 0.5, ())]), 18: lambda: sim.set_device_events(push),
             19: lambda: sim.set_device_terms([])}
    got = []
    for k, f in enumerate(calls):
        if k in setup:
            setup[k]()
        before = sim.launch_count
        try:
            f()
        except WlError:
            assert sim.launch_count == before
            got.append(R)
            continue
        got.append(sim.launch_count - before)
    torch.cuda.synchronize()
    sim.close()
    return got


@pytest.mark.parametrize("config", list(EXPECTED), ids=lambda c: f"{c[0]}-rows{int(c[1])}-events{int(c[2])}")
def test_launches_of_one_call(config):
    got = _launches(*config)
    want = EXPECTED[config]
    diff = {name: (g, w) for name, g, w in zip(CALLS, got, want) if g != w}
    assert not diff, f"launches (got, expected) per call that differs: {diff}; all: {tuple(got)}"
