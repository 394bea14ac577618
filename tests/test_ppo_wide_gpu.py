"""wl_ppo_update_wide (FusedPPO(activation="relu")) against the torch restatement of rsl_rl PPO.update() with ReLU
(tests/ppo_reference_relu.py over tests/ppo_reference.py) run in fp32 and fp64 on the same permutation.
err(x) = ||x - x_fp64|| / ||x_fp64||; the fused update must stay within max(4 * err(torch fp32), 1e-6) of the fp64 run,
each layer's weight and bias taken together."""
import copy
from types import SimpleNamespace

import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")


def _err(x, ref):
    return ((x.double() - ref.double()).norm() / ref.double().norm()).item()


def _nets(D, seed, std=(0.8, 1.2)):
    torch.manual_seed(seed)
    mk = lambda out: torch.nn.Sequential(torch.nn.Linear(D, 64), torch.nn.ReLU(), torch.nn.Linear(64, 64), torch.nn.ReLU(),
                                         torch.nn.Linear(64, out)).to(DEV)
    return mk(2), mk(1), torch.tensor(std, device=DEV)


def _synthetic(D, n, seed=0, edit=None):
    """A batch collected by a perturbed copy of the network (ratios and value changes on both sides of the clips).
    edit(actor, critic) may change the trained network before it is packed."""
    from wheeledlab_b200.policy import pack_actor_critic
    actor, critic, std = _nets(D, seed)
    g = torch.Generator(device=DEV).manual_seed(seed + 1)
    ap, cp = copy.deepcopy(actor), copy.deepcopy(critic)
    with torch.no_grad():
        for net in (ap, cp):
            for p in net.parameters():
                p.add_(0.15 * p.abs().mean() * torch.randn(p.shape, device=DEV, generator=g))
        if edit is not None:
            edit(actor, critic)
        sp = std * torch.tensor([1.15, 0.9], device=DEV)
        obs = torch.randn(n, D, device=DEV, generator=g)
        mu = ap(obs)
        val = cp(obs).squeeze(-1) + 0.25 * torch.randn(n, device=DEV, generator=g)
        act = mu + sp * torch.randn(n, 2, device=DEV, generator=g)
        lp = torch.distributions.Normal(mu, sp).log_prob(act).sum(-1)
        ret = val + 0.5 * torch.randn(n, device=DEV, generator=g)
        adv = 0.3 + torch.randn(n, device=DEV, generator=g)
    blob = pack_actor_critic(actor, critic, std, D, DEV)
    slab = SimpleNamespace(obs_in=obs.contiguous(), actions=act.contiguous(), values=val.contiguous(), log_prob=lp.contiguous(),
                           mean=mu.contiguous())
    perm = torch.randperm(n, device=DEV, generator=g)
    return blob, slab, ret.contiguous(), adv.contiguous(), perm


def _references(blob0, D, slab, ret, adv, perm, cfg, keep_grads=False):
    from ppo_reference_relu import torch_ppo
    out = {}
    for dt in (torch.float32, torch.float64):
        r = torch_ppo(blob0, D, cfg, dt, "relu")
        stats = r.update(slab.obs_in, slab.actions, slab.values, slab.log_prob, slab.mean, ret, adv, perm, keep_grads=keep_grads)
        out[dt] = (r, stats)
    return out[torch.float32], out[torch.float64]


def _layers(g):
    """{layer: weight and bias flattened together} of an rsl_rl state dict (std on its own)."""
    out = {f"{net}.{k}": torch.cat([g[f"{net}.{k}.weight"].reshape(-1), g[f"{net}.{k}.bias"].reshape(-1)])
           for net in ("actor", "critic") for k in (0, 2, 4)}
    out["std"] = g["std"]
    return out


def _padding_mask(D):
    from wheeledlab_b200.policy import blob_layout
    off, total = blob_layout(D)
    lens = [D * 64, 64, 4096, 64, 128, 2, D * 64, 64, 4096, 64, 64, 1, 2]
    m = torch.ones(total, dtype=torch.bool)
    for o, k in zip(off, lens):
        m[o:o + k] = False
    return m.to(DEV)


def _check_gradient(D, n, cfg, seed=0, branches=False, edit=None):
    from wheeledlab_b200.learner import FusedPPO
    from wheeledlab_b200.policy import actor_critic_state_dict
    blob, slab, ret, adv, perm = _synthetic(D, n, seed, edit)
    (r32, s32), (r64, s64) = _references(blob.clone(), D, slab, ret, adv, perm, cfg, keep_grads=True)
    ppo = FusedPPO(blob, D, cfg, activation="relu")
    out = ppo.update(slab, ret, adv, perm)
    torch.cuda.synchronize()
    t = r64.trace[-1]
    if branches:
        ratio, A, lo, hi = t["ratio"], t["A"], 1 - cfg.clip_param, 1 + cfg.clip_param
        for name, sel in (("ratio > 1+clip, A > 0", (ratio > hi) & (A > 0)), ("ratio > 1+clip, A < 0", (ratio > hi) & (A < 0)),
                          ("ratio < 1-clip, A > 0", (ratio < lo) & (A > 0)), ("ratio < 1-clip, A < 0", (ratio < lo) & (A < 0)),
                          ("ratio inside the clip range", (ratio >= lo) & (ratio <= hi)),
                          ("value clipped", t["dv"].abs() > cfg.clip_param), ("value unclipped", t["dv"].abs() <= cfg.clip_param),
                          ("clipped value loss larger", t["vlc"] > t["vl"]), ("plain value loss larger", t["vl"] > t["vlc"])):
            assert int(sel.sum()) > 100, f"the synthetic batch misses the branch: {name}"
    grad = _layers(actor_critic_state_dict(ppo.last_gradient(), D))
    g32, g64 = _layers(r32.trace[-1]["grads"]), _layers(t["grads"])
    for k in g64:
        ef, et = _err(grad[k], g64[k]), _err(g32[k], g64[k])
        assert ef <= max(4 * et, 1e-6), f"D={D} n={n} d{k}: err {ef:.3g} vs torch fp32 {et:.3g}"
    if cfg.num_learning_epochs * cfg.num_mini_batches == 1:
        for k in ("surrogate", "value_function", "entropy", "kl"):
            got, want = out[k].item(), s64[k]
            assert abs(got - want) <= 1e-5 * abs(want) + 1e-7, f"{k}: {got} vs {want}"
    assert not torch.any(blob[_padding_mask(D)] != 0), "a padding float of the blob moved"
    return ppo, grad, t["grads"]


@pytest.mark.parametrize("D", [689, 1, 3, 5, 31, 65])
def test_one_minibatch_gradient_matches_autograd_on_every_branch(D):
    _need_gpu()
    from wheeledlab_b200.learner import PPOConfig
    _check_gradient(D, 16384, PPOConfig(num_learning_epochs=1, num_mini_batches=1), branches=True)


@pytest.mark.parametrize("D,n,mb", [(100, 4231, 1), (689, 100, 1), (129, 3 * 4231, 3), (689, 2 * 12689, 2)])
def test_gradient_with_partial_tiles_and_k_splits(D, n, mb):
    """Mini-batches of 4231 (133 tiles > 132 SMs: one CTA takes two, the last tile has 7 samples), 100 (4 CTAs) and 12 689;
    widths whose last dW1 tile (64 rows) and last layer-1 K chunk (32) are partial.  The last mini-batch's gradient; the
    fixed schedule keeps a KL near a threshold of the adaptive rule from giving the earlier steps different learning rates."""
    _need_gpu()
    from wheeledlab_b200.learner import PPOConfig
    _check_gradient(D, n, PPOConfig(num_learning_epochs=1, num_mini_batches=mb, schedule="fixed"), seed=D)


def test_exactly_zero_pre_activation_has_zero_gradient():
    """Actor unit 5 and critic unit 9 of layer 1 get zero weights and bias: z == 0 exactly for every sample, and torch's
    threshold_backward gives those units (their W1 columns and b1 entries) a zero gradient."""
    _need_gpu()
    from wheeledlab_b200.learner import PPOConfig

    def edit(actor, critic):
        for net, u in ((actor, 5), (critic, 9)):
            net[0].weight[u].zero_(); net[0].bias[u].zero_()

    _, grad, g64 = _check_gradient(37, 4096, PPOConfig(num_learning_epochs=1, num_mini_batches=1), edit=edit)
    for net, u in (("actor", 5), ("critic", 9)):
        assert torch.all(g64[f"{net}.0.weight"][u] == 0) and g64[f"{net}.0.bias"][u] == 0      # (the reference agrees)
        wb = grad[f"{net}.0"]                                # [W1 (out-major [64, 37]) | b1], flattened
        w, b = wb[:64 * 37].view(64, 37), wb[64 * 37:]
        assert torch.all(w[u] == 0) and b[u] == 0, f"{net} unit {u}: nonzero gradient at z == 0"


def _rollout_batch(n_envs, T, seed):
    import wheeledlab_b200 as wl
    from wheeledlab_b200.learner import compute_returns
    from wheeledlab_b200.policy import FusedPolicyRollout, critic_value, pack_actor_critic
    D = 689
    actor, critic, _ = _nets(D, seed)
    blob = pack_actor_critic(actor, critic, torch.ones(2, device=DEV), D, DEV)
    sim = wl.WheeledSim(wl.elevation_task(num_envs=n_envs, seed=seed), DEV); sim.startup(); sim.reset(None, 0)
    roll = FusedPolicyRollout(sim, blob, T, activation="relu").capture(0)
    slab = roll.run()
    last = critic_value(blob, D, roll.obs0, "relu")
    ret, adv = compute_returns(slab.rewards, slab.values, last, slab.terminated | slab.truncated, 0.99, 0.95, time_outs=slab.truncated)
    perm = torch.randperm(T * n_envs, device=DEV, generator=torch.Generator(device=DEV).manual_seed(seed))
    return blob, slab, ret, adv, perm


def test_full_update_on_an_elevation_rollout_follows_the_lr_sequence():
    _need_gpu()
    from ppo_reference_relu import torch_ppo
    from wheeledlab_b200.learner import FusedPPO, PPOConfig
    from wheeledlab_b200.policy import load_actor_critic_state_dict
    D, cfg = 689, PPOConfig()
    blob, slab, ret, adv, perm = _rollout_batch(4096, 128, seed=3)
    (r32, _), (r64, s64) = _references(blob.clone(), D, slab, ret, adv, perm, cfg)
    ppo = FusedPPO(blob, D, cfg, activation="relu")
    ppo.update(slab, ret, adv, perm)
    hist = ppo.history.cpu()
    lrs = [t["lr"] for t in r64.trace]
    assert len(lrs) == 20
    assert [float(x) for x in hist[:, 1]] == pytest.approx(lrs, rel=1e-6), f"lr sequence {hist[:, 1].tolist()} vs {lrs}"
    obs = slab.obs_in.reshape(-1, D)[:65536]
    fused = torch_ppo(blob, D, cfg, torch.float64, "relu").forward(obs)
    b32 = load_actor_critic_state_dict({k: v.float() for k, v in r32.state_dict().items()}, D, device=DEV)
    t32 = torch_ppo(b32, D, cfg, torch.float64, "relu").forward(obs)
    truth = r64.forward(obs)
    for k, name in enumerate(("mean", "value")):
        ef, et = _err(fused[k], truth[k]), _err(t32[k], truth[k])
        assert ef <= max(4 * et, 1e-6), f"{name} after the update: err {ef:.3g} vs torch fp32 {et:.3g}"
    assert not torch.any(blob[_padding_mask(D)] != 0)


def test_update_is_bit_identical_run_to_run_and_under_graph_replay():
    _need_gpu()
    from wheeledlab_b200.learner import FusedPPO, PPOConfig
    D, cfg = 689, PPOConfig(num_learning_epochs=2, num_mini_batches=3)
    blob0, slab, ret, adv, perm = _synthetic(D, 3 * 4231, seed=4)
    outs = []
    for _ in range(2):
        b = blob0.clone()
        FusedPPO(b, D, cfg, activation="relu").update(slab, ret, adv, perm)
        outs.append(b)
    b = blob0.clone()
    ppo = FusedPPO(b, D, cfg, activation="relu")
    ppo._workspace(perm.numel())
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s), torch.cuda.graph(g, stream=s):
        ppo.update(slab, ret, adv, perm)
    torch.cuda.current_stream().wait_stream(s)
    b.copy_(blob0); ppo.m.zero_(); ppo.v.zero_(); ppo.state.zero_(); ppo.state[0] = cfg.learning_rate
    g.replay()
    torch.cuda.synchronize()
    outs.append(b.clone())
    for k, o in enumerate(outs[1:]):
        assert torch.equal(o.view(torch.int32), outs[0].view(torch.int32)), f"run {k + 1} differs from run 0"


def test_ppo_iteration_relu_on_elevation_graph_equals_eager():
    """PPOIteration(activation="relu"): two iterations captured as one graph each replay vs the same two run eagerly."""
    _need_gpu()
    import wheeledlab_b200 as wl
    from wheeledlab_b200.learner import PPOConfig, PPOIteration
    from wheeledlab_b200.policy import pack_actor_critic
    D, n, T = 689, 256, 16
    cfg = PPOConfig(num_mini_batches=4, num_learning_epochs=2)
    actor, critic, _ = _nets(D, 7)
    res = []
    for capture in (False, True):
        blob = pack_actor_critic(actor, critic, torch.ones(2, device=DEV), D, DEV)
        sim = wl.WheeledSim(wl.elevation_task(num_envs=n, seed=13), DEV); sim.startup(); sim.reset(None, 0)
        it = PPOIteration(sim, blob, cfg, T, activation="relu").start(0, capture=capture)
        stats = []
        for k in range(2):
            perm = torch.randperm(T * n, device=DEV, generator=torch.Generator(device=DEV).manual_seed(k))
            stats.append({key: v.item() for key, v in it.run(perm).items()})
        torch.cuda.synchronize()
        res.append((blob.clone(), it.roll.slab.obs_in.clone(), stats))
    assert torch.equal(res[0][0].view(torch.int32), res[1][0].view(torch.int32)), "blob after two iterations differs"
    assert torch.equal(res[0][1].view(torch.int32), res[1][1].view(torch.int32)), "slab differs"
    assert res[0][2] == res[1][2]


def test_wide_update_argument_errors():
    _need_gpu()
    import ctypes as C
    from wheeledlab_b200._lib import WlPpoBatch, WlPpoParams, lib
    fake = 1 << 20
    batch = WlPpoBatch(*([fake] * 8))
    for D, n, rc_want in ((0, 1024, -1), (4097, 1024, -3), (689, 1022, -1)):
        p = WlPpoParams(D, n, 5, 4, 0.2, 1.0, 0.005, 1.0, 0.01, 1, 1, 0)
        assert lib.wl_ppo_update_wide(C.byref(p), C.byref(batch), fake, fake, fake, fake, fake, 1 << 30, None) == rc_want
        assert lib.wl_ppo_wide_workspace_bytes(D, n, 4) == 0
    assert lib.wl_ppo_wide_workspace_bytes(4096, 1024, 4) > lib.wl_ppo_wide_workspace_bytes(1, 1024, 4) > 0
