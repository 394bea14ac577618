"""wl_ppo_update (learner.FusedPPO) against a torch restatement of rsl_rl PPO.update() (tests/ppo_reference.py), run in fp32
and in fp64 on the same permutation.  err(x) = ||x - x_fp64|| / ||x_fp64|| per tensor; the fused update must stay within
max(4 * err(torch fp32), 1e-6) of the fp64 run."""
import copy
import ctypes as C
from types import SimpleNamespace

import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
D = 14


def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")


def _err(x, ref):
    return ((x.double() - ref.double()).norm() / ref.double().norm()).item()


def _nets(seed, std=(0.8, 1.2)):
    torch.manual_seed(seed)
    mk = lambda out: torch.nn.Sequential(torch.nn.Linear(D, 64), torch.nn.ELU(), torch.nn.Linear(64, 64), torch.nn.ELU(),
                                         torch.nn.Linear(64, out)).to(DEV)
    return mk(2), mk(1), torch.tensor(std, device=DEV)


def _synthetic(n, seed=0):
    """A batch collected by a perturbed copy of the network: ratios fall on both sides of the clip range with both signs of
    A, and value changes on both sides of the value clip."""
    from wheeledlab_b200.policy import pack_actor_critic
    actor, critic, std = _nets(seed)
    blob = pack_actor_critic(actor, critic, std, D, DEV)
    g = torch.Generator(device=DEV).manual_seed(seed + 1)
    ap, cp = copy.deepcopy(actor), copy.deepcopy(critic)
    with torch.no_grad():
        for net in (ap, cp):
            for p in net.parameters():
                p.add_(0.15 * p.abs().mean() * torch.randn(p.shape, device=DEV, generator=g))
        sp = std * torch.tensor([1.15, 0.9], device=DEV)
        obs = torch.randn(n, D, device=DEV, generator=g)
        mu = ap(obs)
        val = cp(obs).squeeze(-1) + 0.25 * torch.randn(n, device=DEV, generator=g)     # (the value clip is 0.2)
        act = mu + sp * torch.randn(n, 2, device=DEV, generator=g)
        lp = torch.distributions.Normal(mu, sp).log_prob(act).sum(-1)
        ret = val + 0.5 * torch.randn(n, device=DEV, generator=g)
        adv = 0.3 + torch.randn(n, device=DEV, generator=g)
    slab = SimpleNamespace(obs_in=obs.contiguous(), actions=act.contiguous(), values=val.contiguous(), log_prob=lp.contiguous(),
                           mean=mu.contiguous())
    perm = torch.randperm(n, device=DEV, generator=g)
    return blob, slab, ret.contiguous(), adv.contiguous(), perm


def _references(blob0, slab, ret, adv, perm, cfg, keep_grads=False):
    from ppo_reference import TorchPPO
    out = {}
    for dt in (torch.float32, torch.float64):
        r = TorchPPO(blob0, D, cfg, dt)
        stats = r.update(slab.obs_in, slab.actions, slab.values, slab.log_prob, slab.mean, ret, adv, perm, keep_grads=keep_grads)
        out[dt] = (r, stats)
    return out[torch.float32], out[torch.float64]


def _check_outputs(blob, ref32, ref64, obs, what):
    """actor mean and critic value on obs: fused weights vs fp32 torch weights, both against the fp64 run (evaluated in fp64)."""
    from ppo_reference import TorchPPO
    fused = TorchPPO(blob, D, ref64.cfg, torch.float64).forward(obs)
    t32 = TorchPPO(_to_blob(ref32), D, ref64.cfg, torch.float64).forward(obs)
    truth = ref64.forward(obs)
    for k, name in enumerate(("mean", "value")):
        ef, et = _err(fused[k], truth[k]), _err(t32[k], truth[k])
        assert ef <= max(4 * et, 1e-6), f"{what}: {name} err {ef:.3g} vs torch fp32 {et:.3g}"


def _to_blob(ref):
    from wheeledlab_b200.policy import load_actor_critic_state_dict
    return load_actor_critic_state_dict({k: v.float() for k, v in ref.state_dict().items()}, D, device=DEV)


def _padding_mask(obs_dim=D):
    from wheeledlab_b200.policy import blob_layout
    off, total = blob_layout(obs_dim)
    lens = [obs_dim * 64, 64, 4096, 64, 128, 2, obs_dim * 64, 64, 4096, 64, 64, 1, 2]
    m = torch.ones(total, dtype=torch.bool)
    for o, n in zip(off, lens):
        m[o:o + n] = False
    return m.to(DEV)


def test_one_minibatch_gradient_matches_autograd_on_every_branch():
    _need_gpu()
    from wheeledlab_b200.learner import FusedPPO, PPOConfig
    from wheeledlab_b200.policy import actor_critic_state_dict
    n = 16384
    blob, slab, ret, adv, perm = _synthetic(n)
    cfg = PPOConfig(num_learning_epochs=1, num_mini_batches=1)
    (r32, s32), (r64, s64) = _references(blob.clone(), slab, ret, adv, perm, cfg, keep_grads=True)
    ppo = FusedPPO(blob, D, cfg)
    out = ppo.update(slab, ret, adv, perm)
    torch.cuda.synchronize()
    t = r64.trace[0]
    ratio, A, lo, hi = t["ratio"], t["A"], 1 - cfg.clip_param, 1 + cfg.clip_param
    for name, sel in (("ratio > 1+clip, A > 0", (ratio > hi) & (A > 0)), ("ratio > 1+clip, A < 0", (ratio > hi) & (A < 0)),
                      ("ratio < 1-clip, A > 0", (ratio < lo) & (A > 0)), ("ratio < 1-clip, A < 0", (ratio < lo) & (A < 0)),
                      ("ratio inside the clip range (tie)", (ratio >= lo) & (ratio <= hi)),
                      ("value clipped", t["dv"].abs() > cfg.clip_param), ("value unclipped", t["dv"].abs() <= cfg.clip_param),
                      ("clipped value loss larger", t["vlc"] > t["vl"]), ("plain value loss larger", t["vl"] > t["vlc"])):
        assert int(sel.sum()) > 100, f"the synthetic batch misses the branch: {name}"
    grad = actor_critic_state_dict(ppo.last_gradient(), D)
    g32, g64 = r32.trace[0]["grads"], t["grads"]
    for k in g64:
        ef, et = _err(grad[k], g64[k]), _err(g32[k], g64[k])
        assert ef <= max(4 * et, 1e-6), f"d{k}: err {ef:.3g} vs torch fp32 {et:.3g}"
    for k in ("surrogate", "value_function", "entropy", "kl"):
        got, want = out[k].item(), s64[k]
        assert abs(got - want) <= 1e-5 * abs(want) + 1e-7, f"{k}: {got} vs {want}"
    assert not torch.any(blob[_padding_mask()] != 0)


def _rollout_batch(n_envs, T, seed):
    import wheeledlab_b200 as wl
    from wheeledlab_b200.learner import compute_returns
    from wheeledlab_b200.policy import FusedPolicyRollout, critic_value, pack_actor_critic
    actor, critic, _ = _nets(seed)
    blob = pack_actor_critic(actor, critic, torch.ones(2, device=DEV), D, DEV)       # init_noise_std = 1.0
    sim = wl.WheeledSim(wl.drift_task(num_envs=n_envs, seed=seed), DEV); sim.startup(); sim.reset(None, 0)
    roll = FusedPolicyRollout(sim, blob, T).capture(0)
    slab = roll.run()
    last = critic_value(blob, D, roll.obs0)
    ret, adv = compute_returns(slab.rewards, slab.values, last, slab.terminated | slab.truncated, 0.99, 0.95, time_outs=slab.truncated)
    perm = torch.randperm(T * n_envs, device=DEV, generator=torch.Generator(device=DEV).manual_seed(seed))
    return blob, slab, ret, adv, perm


def test_full_update_at_reference_sizes_follows_the_lr_sequence():
    _need_gpu()
    from wheeledlab_b200.learner import FusedPPO, PPOConfig
    cfg = PPOConfig()
    blob, slab, ret, adv, perm = _rollout_batch(4096, 128, seed=3)
    (r32, _), (r64, s64) = _references(blob.clone(), slab, ret, adv, perm, cfg)
    ppo = FusedPPO(blob, D, cfg)
    out = ppo.update(slab, ret, adv, perm)
    hist = ppo.history.cpu()
    kls = [t["kl"] for t in r64.trace]
    for kl in kls:                                      # the seed keeps every KL clear of the schedule's thresholds
        for thr in (2 * cfg.desired_kl, cfg.desired_kl / 2):
            assert abs(kl - thr) > 1e-3 * thr, f"KL {kl} within 1e-3 of {thr}: pick another seed"
    lrs = torch.tensor([t["lr"] for t in r64.trace], dtype=torch.float64)
    assert torch.allclose(hist[:, 1].double(), lrs, rtol=1e-6, atol=0), (hist[:, 1], lrs)
    assert len(set(lrs.tolist())) > 1, "the lr never moved"
    assert torch.allclose(hist[:, 0].double(), torch.tensor(kls, dtype=torch.float64), rtol=1e-3, atol=1e-7)
    assert abs(out["learning_rate"].item() - s64["learning_rate"]) <= 1e-6 * s64["learning_rate"]
    _check_outputs(blob, r32, r64, slab.obs_in, "4096 x 128, PPOConfig()")
    assert not torch.any(blob[_padding_mask()] != 0) and not torch.any(ppo.m[_padding_mask()] != 0)


@pytest.mark.parametrize("variant", ["fixed", "plain_value_loss", "clip", "no_clip"])
def test_update_variants(variant):
    _need_gpu()
    from wheeledlab_b200.learner import FusedPPO, PPOConfig
    cfg = PPOConfig(num_learning_epochs=2, num_mini_batches=4)
    if variant == "fixed":
        cfg.schedule = "fixed"
    elif variant == "plain_value_loss":
        cfg.use_clipped_value_loss = False
    elif variant == "clip":
        cfg.max_grad_norm = 0.05
    else:
        cfg.max_grad_norm = 1e4
    blob, slab, ret, adv, perm = _synthetic(65536, seed=11)
    (r32, _), (r64, _) = _references(blob.clone(), slab, ret, adv, perm, cfg)
    norms = [t["norm"] for t in r64.trace]
    if variant == "clip":
        assert min(norms) > cfg.max_grad_norm
    if variant == "no_clip":
        assert max(norms) < cfg.max_grad_norm
    ppo = FusedPPO(blob, D, cfg)
    ppo.update(slab, ret, adv, perm)
    lrs = torch.tensor([t["lr"] for t in r64.trace], dtype=torch.float64)
    assert torch.allclose(ppo.history[:, 1].double().cpu(), lrs, rtol=1e-6, atol=0)
    if variant == "fixed":
        assert torch.all(lrs == cfg.learning_rate)
    _check_outputs(blob, r32, r64, slab.obs_in, variant)


def _snapshot(ppo):
    return [x.clone() for x in (ppo.blob, ppo.m, ppo.v, ppo.state)]


def test_update_is_deterministic_and_graph_replay_is_bit_identical():
    _need_gpu()
    from wheeledlab_b200.learner import FusedPPO, PPOConfig
    blob, slab, ret, adv, perm = _synthetic(65536, seed=5)
    cfg = PPOConfig()
    runs = []
    for _ in range(2):
        p = FusedPPO(blob.clone(), D, cfg)
        p.update(slab, ret, adv, perm); p.update(slab, ret, adv, perm)
        runs.append(_snapshot(p))
    g = FusedPPO(blob.clone(), D, cfg)
    g.update(slab, ret, adv, perm)                      # eager first update (sizes the workspace), then a captured one
    graph = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s), torch.cuda.graph(graph, stream=s):
        g.update(slab, ret, adv, perm)
    torch.cuda.current_stream().wait_stream(s)
    graph.replay()
    runs.append(_snapshot(g))
    torch.cuda.synchronize()
    for r in runs[1:]:
        for a, b in zip(runs[0], r):
            assert torch.equal(a.view(torch.int32), b.view(torch.int32))
    assert not torch.any(runs[0][0][_padding_mask()] != 0)


def test_whole_iteration_graph_replays_equal_the_eager_sequence():
    _need_gpu()
    import wheeledlab_b200 as wl
    from wheeledlab_b200.learner import PPOConfig, PPOIteration
    from wheeledlab_b200.policy import pack_actor_critic
    n, T = 2048, 32
    actor, critic, std = _nets(9, std=(1.0, 1.0))
    its = []
    for capture in (False, True):
        sim = wl.WheeledSim(wl.drift_task(num_envs=n, seed=4), DEV); sim.startup(); sim.reset(None, 0)
        blob = pack_actor_critic(actor, critic, std, D, DEV)
        its.append(PPOIteration(sim, blob, PPOConfig(), T).start(0, capture=capture))
    g = torch.Generator(device=DEV).manual_seed(1)
    for k in range(3):
        perm = torch.randperm(n * T, device=DEV, generator=g)
        outs = [it.run(perm) for it in its]
        torch.cuda.synchronize()
        a, b = its
        for x, y in ((a.blob, b.blob), (a.ppo.m, b.ppo.m), (a.ppo.v, b.ppo.v), (a.ppo.state, b.ppo.state),
                     (a.roll.slab.flat, b.roll.slab.flat)):
            assert torch.equal(x.view(torch.uint8), y.view(torch.uint8)), f"iteration {k}"
        assert all(torch.equal(outs[0][key], outs[1][key]) for key in outs[0])
    assert not torch.any(its[1].blob[_padding_mask()] != 0)


def test_argument_errors_name_the_entry_point():
    _need_gpu()
    import wheeledlab_b200 as wl
    from wheeledlab_b200.learner import FusedPPO, PPOConfig
    blob, slab, ret, adv, perm = _synthetic(4096)
    with pytest.raises(wl.WlError, match="wl_ppo_workspace_bytes.*obs_dim"):
        FusedPPO(torch.zeros_like(blob), 17, PPOConfig()).update(slab, ret, adv, perm)
    with pytest.raises(wl.WlError, match="wl_ppo_workspace_bytes.*num_mini_batches"):
        FusedPPO(blob, D, PPOConfig(num_mini_batches=3)).update(slab, ret, adv, perm)
    ppo = FusedPPO(blob, D, PPOConfig())
    ppo.update(slab, ret, adv, perm)
    from wheeledlab_b200._lib import WlPpoBatch, WlPpoParams
    p = WlPpoParams(D, 4096, 1, 4, 0.2, 1.0, 0.005, 1.0, 0.01, 1, 1, 0)
    b = WlPpoBatch(*[x.data_ptr() for x in (slab.obs_in, slab.actions, slab.values, slab.log_prob, slab.mean, ret, adv, perm)])
    ws = ppo.workspace
    call = lambda blob_ptr, nbytes: wl.lib.wl_ppo_update(C.byref(p), C.byref(b), C.c_void_p(blob_ptr), C.c_void_p(ppo.m.data_ptr()),
                                                         C.c_void_p(ppo.v.data_ptr()), C.c_void_p(ppo.state.data_ptr()),
                                                         C.c_void_p(ws.data_ptr()), nbytes, None)
    assert call(blob.data_ptr() + 4, ws.numel()) == -1 and b"d_blob" in wl.lib.wl_last_error()
    assert call(blob.data_ptr(), 1024) == -1 and b"workspace_bytes" in wl.lib.wl_last_error()
