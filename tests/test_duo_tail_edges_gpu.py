"""The Drift duo step kernel's post-physics tail on states at its edges, against the thread-per-env kernel, bit for bit.

The shipped step specs run the tail as selects (euler angles, the reset / push choice, the observation slice, the state stores;
DESIGN.md 6e).  One warp holds eight envs, so every warp here mixes: an exact-zero quaternion at rest, subnormal quaternion
components, |sin_pitch| at and above 1 of both signs, a high- and a low-frequency push firing, and resets with and without a
push due; zero and subnormal body velocities feed the reward tail's roots and slip angle."""
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

G_POS, G_QUAT, G_LINVEL, G_ANGVEL = 0, 1, 2, 3


def _set_edges(sim, max_len):
    g = sim.groups
    n = g.shape[1]
    k = torch.arange(n, device=g.device) % 8
    h = 0.70710678118654752
    quats = torch.tensor([[1.0, 0.0, 0.0, 0.0], [1.0, 1e-40, 1e-41, 0.0], [h, 0.0, h, 0.0], [h, 0.0, -h, 0.0],
                          [0.5, 0.0, 0.70710683, 0.5], [1.0, -2e-39, 0.0, 3e-39], [0.0, 0.0, 1.0, 0.0], [h, 0.0, 0.0, h]],
                         device=g.device)
    g[G_QUAT] = quats[k]
    rest = (k <= 3) | (k == 5)
    g[G_LINVEL, rest, 0:3] = 0.0
    g[G_ANGVEL, rest, 0:3] = 0.0
    g[G_LINVEL, k == 3, 0:3] = torch.tensor([1e-40, -3e-41, 0.0], device=g.device)   # subnormal body velocity
    g[G_LINVEL, (k == 4) | (k == 7), 3] = 0.0          # high-frequency push due this step
    g[G_ANGVEL, (k == 5) | (k == 7), 3] = 0.0          # low-frequency push due this step
    ep = g[G_POS, :, 3].view(torch.int32)
    ep[(k == 6) | (k == 7)] = max_len - 1              # times out (and resets) this step


@pytest.mark.parametrize("task", ["drift", "hound_4wd"])
def test_duo_tail_edges_match_thread_per_env(task):
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import wheeledlab_b200 as wl

    def mk():
        return wl.make_task(task, num_envs=256, seed=11)

    ref, duo = wl.WheeledSim(mk(), "cuda:0"), wl.WheeledSim(mk(), "cuda:0")
    ref.set_kernel_variant(1); duo.set_kernel_variant(8)
    max_len = int(mk().cfg.max_episode_length)
    for s in (ref, duo):
        s.startup(); s.reset(None, 0)
    for t in range(6):
        if t % 3 == 0:
            for s in (ref, duo):
                _set_edges(s, max_len)
        act = ref.synth_actions(t)
        ra, rd = ref.step(act, t), duo.step(act, t)
        for x, y in zip(ra, rd):
            assert torch.equal(x.view(torch.uint8) if x.dtype == torch.float32 else x,
                               y.view(torch.uint8) if y.dtype == torch.float32 else y), f"{task}: outputs differ at step {t}"
        assert torch.equal(ref.groups.view(torch.int32), duo.groups.view(torch.int32)), f"{task}: state differs after step {t}"
        if t % 3 == 0:
            assert int((ra[2] | ra[3]).sum().item()) >= 2 * (256 // 8), "the edge states did not reset"
