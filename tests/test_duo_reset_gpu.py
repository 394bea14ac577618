"""The duo step kernel's auto-reset with interval pushes off.  The aux warp draws every env's reset outcome, push timers
included, and the env warp applies it to the envs that reset; without pushes the fresh timers must be stored as drawn.
No shipped config turns pushes off, so the generic duo body runs this one: identical bits to the thread-per-env kernel."""
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")


def test_duo_reset_without_pushes_matches_thread_per_env():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import wheeledlab_b200 as wl

    def mk():
        spec = wl.make_task("drift", num_envs=4096, seed=5)
        spec.cfg.push_enable = 0
        return spec

    ref, duo = wl.WheeledSim(mk(), "cuda:0"), wl.WheeledSim(mk(), "cuda:0")
    ref.set_kernel_variant(1); duo.set_kernel_variant(8)
    for s in (ref, duo):
        s.startup(); s.reset(None, 0)
    resets = 0
    for t in range(400):
        act = ref.synth_actions(t)
        ra, rd = ref.step(act, t), duo.step(act, t)
        for x, y in zip(ra, rd):
            assert torch.equal(x, y), f"duo and thread-per-env kernels differ at step {t}"
        resets += int((ra[2] | ra[3]).sum().item())
    assert torch.equal(ref.groups, duo.groups) and torch.equal(ref.rew_weight, duo.rew_weight)
    assert resets > 0, "trajectory too short to exercise the auto-reset"
