"""The duo step kernel specialised on a config's step spec (action map, bounding, pushes, noise, sub-step counts fixed at
compile time) against the thread-per-env kernel, which reads every one of those fields at run time: identical bits."""
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")


def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


def _tanh_drift(**kw):
    import wheeledlab_b200 as wl
    from wheeledlab_b200.tasks import BOUND_TANH
    spec = wl.make_task("drift", **kw)
    spec.cfg.bounding = BOUND_TANH               # no specialisation has this spec: the generic duo kernel runs it
    return spec


@pytest.mark.parametrize("task", ["drift", "hound_4wd", "drift_tanh"])
def test_duo_kernel_matches_thread_per_env(task):
    _need_gpu()
    import wheeledlab_b200 as wl
    mk = (lambda: _tanh_drift(num_envs=4096, seed=11)) if task == "drift_tanh" else (lambda: wl.make_task(task, num_envs=4096, seed=11))
    ref, duo = wl.WheeledSim(mk(), "cuda:0"), wl.WheeledSim(mk(), "cuda:0")
    ref.set_kernel_variant(1); duo.set_kernel_variant(8)
    for s in (ref, duo):
        s.startup(); s.reset(None, 0)
    resets = 0
    for t in range(400):
        act = ref.synth_actions(t)
        ra, rd = ref.step(act, t), duo.step(act, t)
        for x, y in zip(ra, rd):
            assert torch.equal(x, y), f"{task}: duo and thread-per-env kernels differ at step {t}"
        resets += int((ra[2] | ra[3]).sum().item())
    assert torch.equal(ref.groups, duo.groups) and torch.equal(ref.rew_weight, duo.rew_weight)
    assert resets > 0, "trajectory too short to exercise the auto-reset"
