"""Consecutive duo-kernel steps of ONE Drift sim, launched with programmatic dependent launch: each step's prologue runs
while the previous step is still finishing, and its griddepcontrol.wait must order every read of the state, the actions
and wl_globals after the previous step's writes.  300 steps on the device-resident counter (the last node advances it)
cross the 250-step curriculum boundary with auto-resets, in one CUDA graph and as eager stream launches; every output and
the final state must match the thread-per-env kernel bit for bit."""
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

N, K = 4096, 300


def _drift():
    import wheeledlab_b200 as wl
    spec = wl.make_task("drift", num_envs=N, seed=13)
    for k in range(spec.cfg.curr_n):
        spec.cfg.curr_every[k] = 1               # every term's weight moves at the first boundary (t = 250)
    return spec


@pytest.mark.parametrize("mode", ["graph", "eager"])
def test_pdl_chained_duo_steps_match_thread_per_env(mode):
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from wheeledlab_b200 import WheeledSim
    dev = "cuda:0"
    ref, duo = WheeledSim(_drift(), dev), WheeledSim(_drift(), dev)
    ref.set_kernel_variant(1); duo.set_kernel_variant(8)
    for s in (ref, duo):
        s.startup(); s.reset(None, 0)
    w0 = ref.rew_weight.clone()
    acts = torch.stack([ref.synth_actions(t) for t in range(K)])
    obs = torch.empty((K, N, duo.obs_dim), dtype=torch.float32, device=dev)
    rew = torch.empty((K, N), dtype=torch.float32, device=dev)
    term = torch.empty((K, N), dtype=torch.uint8, device=dev)
    trunc = torch.empty((K, N), dtype=torch.uint8, device=dev)

    def body():
        for k in range(K):
            duo.step(acts[k], WheeledSim.device_counter_plus(k), out=(obs[k], rew[k], term[k], trunc[k]))
        duo.advance_counter(K)

    duo.set_step_counter(0)
    if mode == "graph":
        g, s = torch.cuda.CUDAGraph(), torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            with torch.cuda.graph(g, stream=s):
                body()
        torch.cuda.current_stream().wait_stream(s)
        duo.set_step_counter(0)                  # (capture moved the host mirror only)
        g.replay()
    else:
        body()
    torch.cuda.synchronize()

    resets = 0
    for t in range(K):
        ro, rr, rt, ru = ref.step(acts[t], t)
        assert torch.equal(ro, obs[t]) and torch.equal(rr, rew[t]), f"{mode}: observation / reward differ at step {t}"
        assert torch.equal(rt, term[t]) and torch.equal(ru, trunc[t]), f"{mode}: done masks differ at step {t}"
        resets += int((rt | ru).sum().item())
    assert torch.equal(ref.groups, duo.groups), f"{mode}: final state differs"
    assert torch.equal(ref.rew_weight, duo.rew_weight), f"{mode}: reward weights differ after the curriculum boundary"
    assert not torch.equal(ref.rew_weight, w0), "the curriculum boundary did not move the weights"
    assert resets > 0, "trajectory too short to exercise the auto-reset"
