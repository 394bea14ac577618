"""wl_ppo_update (learner.FusedPPO) off the one shape test_ppo_update_gpu runs it at (obs_dim 14, mini-batches of whole
32-sample tiles, >= 128 tiles, <= 256 updates), against the same fp32 / fp64 torch restatement (tests/ppo_reference.py)
on the same permutation and with the same criterion: err(x) = ||x - x_fp64|| / ||x_fp64|| per tensor, and the fused update
must stay within max(4 * err(torch fp32), 1e-6) of the fp64 run.

- obs_dim 1..16: the grad kernel's `i1 + k < D` row guard, the (D + 3) & ~3 first-layer width, the zero-filled observation
  columns, and ppo_is_param on the padded W1 rows.
- Mini-batch sizes that end in a partial 32-sample tile, with fewer tiles than SMs, and with one CTA taking two tiles.
- More than WL_PPO_MAX_UPDATES (256) mini-batches: the history is capped and the later rows are not written.
- Rollout batches of the other Drift-family tasks and of the blind Visual task (obs_dim 8) through PPOIteration.
- Process state: updates of different obs_dim in one process, and a process whose first update is captured in a graph
  (child processes, so that earlier tests in this process cannot set the kernel attributes first)."""
import copy
import os
import subprocess
import sys
from pathlib import Path
from types import SimpleNamespace

import pytest

ROOT = Path(__file__).resolve().parent.parent
if __name__ == "__main__":                                  # the child processes of the process-state tests
    sys.path[:0] = [str(ROOT), str(ROOT / "tests")]

torch = pytest.importorskip("torch")

DEV = "cuda:0"
OBS_DIMS = [1, 3, 4, 5, 8, 12, 13, 16]


def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")


def _err(x, ref):
    return ((x.double() - ref.double()).norm() / ref.double().norm()).item()


def _within(ef, et):
    return ef <= max(4 * et, 1e-6)


def _nets(seed, obs_dim, std=(0.8, 1.2)):
    torch.manual_seed(seed)
    mk = lambda out: torch.nn.Sequential(torch.nn.Linear(obs_dim, 64), torch.nn.ELU(), torch.nn.Linear(64, 64), torch.nn.ELU(),
                                         torch.nn.Linear(64, out)).to(DEV)
    return mk(2), mk(1), torch.tensor(std, device=DEV)


def _synthetic(n, obs_dim, seed=0):
    """test_ppo_update_gpu._synthetic at any obs_dim: a batch collected by a perturbed copy of the network, so ratios fall
    on both sides of the clip range with both signs of A, and value changes on both sides of the value clip."""
    from wheeledlab_b200.policy import pack_actor_critic
    actor, critic, std = _nets(seed, obs_dim)
    blob = pack_actor_critic(actor, critic, std, obs_dim, DEV)
    g = torch.Generator(device=DEV).manual_seed(seed + 1)
    ap, cp = copy.deepcopy(actor), copy.deepcopy(critic)
    with torch.no_grad():
        for net in (ap, cp):
            for p in net.parameters():
                p.add_(0.15 * p.abs().mean() * torch.randn(p.shape, device=DEV, generator=g))
        sp = std * torch.tensor([1.15, 0.9], device=DEV)
        obs = torch.randn(n, obs_dim, device=DEV, generator=g)
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


def _references(blob0, obs_dim, slab, ret, adv, perm, cfg, keep_grads=False):
    from ppo_reference import TorchPPO
    out = {}
    for dt in (torch.float32, torch.float64):
        r = TorchPPO(blob0, obs_dim, cfg, dt)
        stats = r.update(slab.obs_in, slab.actions, slab.values, slab.log_prob, slab.mean, ret, adv, perm, keep_grads=keep_grads)
        out[dt] = (r, stats)
    return out[torch.float32], out[torch.float64]


def _to_blob(ref, obs_dim):
    from wheeledlab_b200.policy import load_actor_critic_state_dict
    return load_actor_critic_state_dict({k: v.float() for k, v in ref.state_dict().items()}, obs_dim, device=DEV)


def _check_outputs(blob, obs_dim, ref32, ref64, obs, what):
    """actor mean and critic value on obs: fused weights vs fp32 torch weights, both against the fp64 run (evaluated in fp64)."""
    from ppo_reference import TorchPPO
    fused = TorchPPO(blob, obs_dim, ref64.cfg, torch.float64).forward(obs)
    t32 = TorchPPO(_to_blob(ref32, obs_dim), obs_dim, ref64.cfg, torch.float64).forward(obs)
    truth = ref64.forward(obs)
    for k, name in enumerate(("mean", "value")):
        ef, et = _err(fused[k], truth[k]), _err(t32[k], truth[k])
        assert _within(ef, et), f"{what}: {name} err {ef:.3g} vs torch fp32 {et:.3g}"


def _check_gradient(ppo, obs_dim, r32, r64, what, k=-1):
    """Per layer, (weight, bias) together, and std: a bias gradient is a sum over the batch that can cancel to a small part
    of its usual size (at B = 32 * 132 * 3 + 17 the critic head's bias gradient came out 60x smaller than at another seed,
    with the same absolute error), so it is measured against its layer's gradient norm."""
    from wheeledlab_b200.policy import actor_critic_state_dict
    grad = actor_critic_state_dict(ppo.last_gradient(), obs_dim)
    g32, g64 = r32.trace[k]["grads"], r64.trace[k]["grads"]
    groups = [[f"{net}.{i}.weight", f"{net}.{i}.bias"] for net in ("actor", "critic") for i in (0, 2, 4)] + [["std"]]
    assert sorted(sum(groups, [])) == sorted(g64)
    cat = lambda g, names: torch.cat([g[x].double().reshape(-1) for x in names])
    for names in groups:
        ref = cat(g64, names)
        ef, et = _err(cat(grad, names), ref), _err(cat(g32, names), ref)
        assert _within(ef, et), f"{what}: d{names} err {ef:.3g} vs torch fp32 {et:.3g}"


def _padding_mask(obs_dim):
    from wheeledlab_b200.policy import blob_layout
    off, total = blob_layout(obs_dim)
    lens = [obs_dim * 64, 64, 4096, 64, 128, 2, obs_dim * 64, 64, 4096, 64, 64, 1, 2]
    m = torch.ones(total, dtype=torch.bool)
    for o, n in zip(off, lens):
        m[o:o + n] = False
    return m.to(DEV)


def _check_padding(ppo, obs_dim, what):
    mask = _padding_mask(obs_dim)
    for name, x in (("blob", ppo.blob), ("Adam m", ppo.m), ("Adam v", ppo.v)):
        assert not torch.any(x[mask] != 0), f"{what}: {name} padding is not zero"


# ---- obs_dim -----------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("obs_dim", OBS_DIMS)
def test_gradient_and_update_at_every_obs_dim(obs_dim):
    """One mini-batch's gradient against autograd with every branch of the loss populated, then 2 epochs x 4 mini-batches."""
    _need_gpu()
    from wheeledlab_b200.learner import FusedPPO, PPOConfig
    n = 16384
    blob, slab, ret, adv, perm = _synthetic(n, obs_dim, seed=obs_dim)
    cfg = PPOConfig(num_learning_epochs=1, num_mini_batches=1)
    (r32, _), (r64, s64) = _references(blob.clone(), obs_dim, slab, ret, adv, perm, cfg, keep_grads=True)
    ppo = FusedPPO(blob.clone(), obs_dim, cfg)
    out = ppo.update(slab, ret, adv, perm)
    torch.cuda.synchronize()
    t = r64.trace[0]
    ratio, A, lo, hi = t["ratio"], t["A"], 1 - cfg.clip_param, 1 + cfg.clip_param
    for name, sel in (("ratio > 1+clip, A > 0", (ratio > hi) & (A > 0)), ("ratio > 1+clip, A < 0", (ratio > hi) & (A < 0)),
                      ("ratio < 1-clip, A > 0", (ratio < lo) & (A > 0)), ("ratio < 1-clip, A < 0", (ratio < lo) & (A < 0)),
                      ("ratio inside the clip range (tie)", (ratio >= lo) & (ratio <= hi)),
                      ("value clipped", t["dv"].abs() > cfg.clip_param), ("value unclipped", t["dv"].abs() <= cfg.clip_param),
                      ("clipped value loss larger", t["vlc"] > t["vl"]), ("plain value loss larger", t["vl"] > t["vlc"])):
        assert int(sel.sum()) > 100, f"obs_dim {obs_dim}: the synthetic batch misses the branch: {name}"
    _check_gradient(ppo, obs_dim, r32, r64, f"obs_dim {obs_dim}")
    for k in ("surrogate", "value_function", "entropy", "kl"):
        got, want = out[k].item(), s64[k]
        assert abs(got - want) <= 1e-5 * abs(want) + 1e-7, f"obs_dim {obs_dim}: {k}: {got} vs {want}"
    _check_padding(ppo, obs_dim, f"obs_dim {obs_dim}, one mini-batch")

    cfg = PPOConfig(num_learning_epochs=2, num_mini_batches=4)
    (r32, _), (r64, s64) = _references(blob.clone(), obs_dim, slab, ret, adv, perm, cfg)
    ppo = FusedPPO(blob.clone(), obs_dim, cfg)
    out = ppo.update(slab, ret, adv, perm)
    lrs = torch.tensor([x["lr"] for x in r64.trace], dtype=torch.float64)
    assert torch.allclose(ppo.history[:, 1].double().cpu(), lrs, rtol=1e-6, atol=0)
    _check_outputs(ppo.blob, obs_dim, r32, r64, slab.obs_in, f"obs_dim {obs_dim}, 2 x 4 mini-batches")
    _check_padding(ppo, obs_dim, f"obs_dim {obs_dim}, 2 x 4 mini-batches")


# ---- mini-batch shapes ---------------------------------------------------------------------------------------------------
def _batch_sizes():
    """(name, B): a 1-sample tail tile; a partial tile with fewer CTAs than SMs; one CTA taking two tiles, the second
    partial; exact multiples of the tile with one CTA per SM plus one; three tiles per SM and a 17-sample tail."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count if torch.cuda.is_available() else 132
    return [("33", 33), ("1000", 1000), ("32sms+1", 32 * sms + 1), ("32(sms+1)", 32 * (sms + 1)), ("96sms+17", 32 * sms * 3 + 17)]


@pytest.mark.gpu
@pytest.mark.parametrize("num_mini_batches", [1, 3])
@pytest.mark.parametrize("shape", [s for s, _ in _batch_sizes()])
def test_mini_batch_shapes(shape, num_mini_batches):
    """Mini-batch B, batch = B x num_mini_batches: with 3 mini-batches the row0 offsets of the later ones are not multiples of
    32.  The first mini-batch's gradient against autograd, then a 2-epoch update's outputs and padding."""
    _need_gpu()
    from wheeledlab_b200.learner import FusedPPO, PPOConfig
    D = 14
    B = dict(_batch_sizes())[shape]
    n = B * num_mini_batches
    blob, slab, ret, adv, perm = _synthetic(n, D, seed=B + num_mini_batches)
    what = f"B={B} x {num_mini_batches}"
    cfg = PPOConfig(num_learning_epochs=1, num_mini_batches=1)          # the gradient of one whole mini-batch of B
    sub = SimpleNamespace(**{k: getattr(slab, k)[:B].contiguous() for k in ("obs_in", "actions", "values", "log_prob", "mean")})
    sperm = torch.randperm(B, device=DEV, generator=torch.Generator(device=DEV).manual_seed(B))
    (r32, _), (r64, _) = _references(blob.clone(), D, sub, ret[:B].contiguous(), adv[:B].contiguous(), sperm, cfg, keep_grads=True)
    ppo = FusedPPO(blob.clone(), D, cfg)
    ppo.update(sub, ret[:B].contiguous(), adv[:B].contiguous(), sperm)
    _check_gradient(ppo, D, r32, r64, what)

    cfg = PPOConfig(num_learning_epochs=2, num_mini_batches=num_mini_batches)
    (r32, _), (r64, s64) = _references(blob.clone(), D, slab, ret, adv, perm, cfg)
    ppo = FusedPPO(blob.clone(), D, cfg)
    out = ppo.update(slab, ret, adv, perm)
    lrs = torch.tensor([x["lr"] for x in r64.trace], dtype=torch.float64)
    assert torch.allclose(ppo.history[:, 1].double().cpu(), lrs, rtol=1e-6, atol=0), what
    assert abs(out["learning_rate"].item() - s64["learning_rate"]) <= 1e-6 * s64["learning_rate"], what
    _check_outputs(ppo.blob, D, r32, r64, slab.obs_in, what)
    _check_padding(ppo, D, what)


# ---- more than WL_PPO_MAX_UPDATES mini-batches ---------------------------------------------------------------------------
@pytest.mark.gpu
def test_more_updates_than_the_history_holds():
    """65 epochs x 4 mini-batches = 260 updates.  desired_kl is far below every KL, so the adaptive rule divides the lr by
    1.5 at each update down to its 1e-5 floor (a moving lr no fp32 rounding can flip).  The history keeps the first 256
    (KL, lr) pairs; the last 4 updates must leave them alone."""
    _need_gpu()
    from wheeledlab_b200._lib import lib
    from wheeledlab_b200.learner import FusedPPO, PPOConfig
    D, n = 14, 4096
    cap = (lib.wl_ppo_state_floats() - 10) // 2
    assert cap == 256
    cfg = PPOConfig(num_learning_epochs=65, num_mini_batches=4, desired_kl=1e-9)
    blob, slab, ret, adv, perm = _synthetic(n, D, seed=7)
    (r32, _), (r64, s64) = _references(blob.clone(), D, slab, ret, adv, perm, cfg)
    ppo = FusedPPO(blob.clone(), D, cfg)
    out = ppo.update(slab, ret, adv, perm)
    hist = ppo.history.cpu().double()
    assert hist.shape == (cap, 2)
    kl64 = torch.tensor([x["kl"] for x in r64.trace], dtype=torch.float64)
    kl32 = torch.tensor([x["kl"] for x in r32.trace], dtype=torch.float64)
    lrs = torch.tensor([x["lr"] for x in r64.trace], dtype=torch.float64)
    assert len(kl64) == 260 and min(kl64) > 2 * cfg.desired_kl
    # the first rows hold lr 1e-3 / 1.5^(k+1) and the last updates run at the 1e-5 floor: a later update that wrapped
    # around into the first rows would show in the lr column
    assert len(set(lrs[:8].tolist())) == 8 and lrs[-1] == 1e-5
    assert torch.allclose(hist[:, 1], lrs[:cap], rtol=1e-6, atol=0)
    # each KL against the fp64 run, within 4x torch fp32's own error on that mini-batch (or 1e-4 relative)
    tol = torch.maximum(4 * (kl32[:cap] - kl64[:cap]).abs(), 1e-4 * kl64[:cap].abs())
    bad = ((hist[:, 0] - kl64[:cap]).abs() > tol).nonzero().flatten().tolist()
    assert not bad, f"history KL rows {bad[:8]} differ from the fp64 run"
    assert abs(out["learning_rate"].item() - s64["learning_rate"]) <= 1e-6 * s64["learning_rate"]
    assert abs(out["kl"].item() - s64["kl"]) <= max(4 * abs(r32.trace[-1]["kl"] - s64["kl"]), 1e-4 * s64["kl"])
    _check_outputs(ppo.blob, D, r32, r64, slab.obs_in, "260 updates")
    _check_padding(ppo, D, "260 updates")


# ---- rollout batches of the other tasks ----------------------------------------------------------------------------------
def _task_spec(name, n, seed):
    import wheeledlab_b200 as wl
    if name == "visual":
        return wl.visual_task(num_envs=n, seed=seed)               # blind: obs_dim 8
    return wl.make_task(name, num_envs=n, seed=seed)


@pytest.mark.gpu
@pytest.mark.parametrize("task", ["hound_4wd", "f1tenth_drift", "visual"])
def test_iteration_on_other_tasks(task):
    """PPOIteration eager and captured: bit-identical over 3 iterations; the first update matches TorchPPO on the
    rollout the iteration collected."""
    _need_gpu()
    import wheeledlab_b200 as wl
    from wheeledlab_b200.learner import PPOConfig, PPOIteration, compute_returns
    from wheeledlab_b200.policy import critic_value, pack_actor_critic
    n, T = 1024, 32
    cfg = PPOConfig()
    its, blob0 = [], None
    for capture in (False, True):
        sim = wl.WheeledSim(_task_spec(task, n, 4), DEV); sim.startup(); sim.reset(None, 0)
        D = sim.obs_dim
        actor, critic, std = _nets(9, D, std=(1.0, 1.0))
        blob = pack_actor_critic(actor, critic, std, D, DEV)
        blob0 = blob.clone()
        its.append(PPOIteration(sim, blob, cfg, T).start(0, capture=capture))
    assert D == (8 if task == "visual" else 14)
    g = torch.Generator(device=DEV).manual_seed(1)
    for k in range(3):
        perm = torch.randperm(n * T, device=DEV, generator=g)
        outs = [it.run(perm) for it in its]
        torch.cuda.synchronize()
        a, b = its
        for x, y in ((a.blob, b.blob), (a.ppo.m, b.ppo.m), (a.ppo.v, b.ppo.v), (a.ppo.state, b.ppo.state),
                     (a.roll.slab.flat, b.roll.slab.flat)):
            assert torch.equal(x.view(torch.uint8), y.view(torch.uint8)), f"{task}: iteration {k}"
        assert all(torch.equal(outs[0][key], outs[1][key]) for key in outs[0])
        if k == 0:                                           # the first update against the references on the same rollout
            slab = a.roll.slab
            last = critic_value(blob0, D, a.roll.obs0)
            ret, adv = compute_returns(slab.rewards, slab.values, last, slab.terminated | slab.truncated, cfg.gamma, cfg.lam,
                                       time_outs=slab.truncated)
            (r32, _), (r64, s64) = _references(blob0.clone(), D, slab, ret, adv, perm, cfg)
            _check_outputs(a.blob, D, r32, r64, slab.obs_in, f"{task}: first update")
    _check_padding(its[1].ppo, D, task)


# ---- process state (child processes) -------------------------------------------------------------------------------------
def _child_mixed_obs_dims():
    """Updates of obs_dim 8, then 14, then 4 in one process, each against the references."""
    from wheeledlab_b200.learner import FusedPPO, PPOConfig
    cfg = PPOConfig(num_learning_epochs=2, num_mini_batches=4)
    for D in (8, 14, 4):
        blob, slab, ret, adv, perm = _synthetic(8192, D, seed=D)
        (r32, _), (r64, _) = _references(blob.clone(), D, slab, ret, adv, perm, cfg)
        ppo = FusedPPO(blob, D, cfg)
        ppo.update(slab, ret, adv, perm)
        _check_outputs(ppo.blob, D, r32, r64, slab.obs_in, f"obs_dim {D} after earlier obs_dims")
        _check_padding(ppo, D, f"obs_dim {D}")


def _child_first_update_captured():
    """The first act step and the first wl_ppo_update of the process are recorded inside PPOIteration.start(capture=True);
    its replays must equal an eager iteration's results."""
    import wheeledlab_b200 as wl
    from wheeledlab_b200.learner import PPOConfig, PPOIteration
    from wheeledlab_b200.policy import pack_actor_critic
    n, T = 512, 16
    its = []
    for capture in (True, False):
        sim = wl.WheeledSim(wl.drift_task(num_envs=n, seed=6), DEV); sim.startup(); sim.reset(None, 0)
        actor, critic, std = _nets(2, 14, std=(1.0, 1.0))
        its.append(PPOIteration(sim, pack_actor_critic(actor, critic, std, 14, DEV), PPOConfig(), T).start(0, capture=capture))
    g = torch.Generator(device=DEV).manual_seed(3)
    for k in range(2):
        perm = torch.randperm(n * T, device=DEV, generator=g)
        for it in its:
            it.run(perm)
        torch.cuda.synchronize()
        a, b = its
        for x, y in ((a.blob, b.blob), (a.ppo.state, b.ppo.state), (a.roll.slab.flat, b.roll.slab.flat)):
            assert torch.equal(x.view(torch.uint8), y.view(torch.uint8)), f"iteration {k}"
    assert torch.isfinite(its[0].blob).all()


def _run_child(which):
    r = subprocess.run([sys.executable, str(Path(__file__).resolve()), which], capture_output=True, text=True, timeout=600,
                       cwd=str(ROOT), env=dict(os.environ))
    assert r.returncode == 0, f"{which}:\n{r.stdout[-2000:]}\n{r.stderr[-4000:]}"


@pytest.mark.gpu
def test_updates_of_different_obs_dim_in_one_process():
    """The grad kernel's shared memory grows with obs_dim; its per-device limit must hold the widest obs_dim whatever the
    first update in the process was."""
    _need_gpu()
    _run_child("mixed_obs_dims")


@pytest.mark.gpu
def test_first_update_of_the_process_inside_a_graph_capture():
    _need_gpu()
    _run_child("first_update_captured")


if __name__ == "__main__":
    {"mixed_obs_dims": _child_mixed_obs_dims, "first_update_captured": _child_first_update_captured}[sys.argv[1]]()
    print("ok")
