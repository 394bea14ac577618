"""The data-parallel PPO update (wl_ppo_update_dp, DESIGN 6j) on one GPU.  R = 1 is wl_ppo_update / wl_ppo_update_wide bit
for bit; R emulated ranks in one process (every rank local, one stream) keep bit-identical replicas and follow a torch
restatement of rsl_rl's multi-GPU PPO.update() within max(4 * err(torch fp32), 1e-6) of its fp64 run; env shards
concatenate to one big rollout; a captured one-process iteration replays as the eager sequence."""
import copy
from types import SimpleNamespace

import pytest
import torch
from torch import nn

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")


def _err(x, ref):
    return ((x.double() - ref.double()).norm() / ref.double().norm()).item()


def _nets(D, activation, seed, std=(0.8, 1.2)):
    torch.manual_seed(seed)
    act = nn.ELU if activation == "elu" else nn.ReLU
    mk = lambda out: nn.Sequential(nn.Linear(D, 64), act(), nn.Linear(64, 64), act(), nn.Linear(64, out)).to(DEV)
    return mk(2), mk(1), torch.tensor(std, device=DEV)


def _batch(actor, critic, std, D, n, g):
    """Rows collected by a perturbed copy of the network (ratios on both sides of the clip range, values on both sides
    of the value clip), as tests/test_ppo_update_gpu.py draws them."""
    ap, cp = copy.deepcopy(actor), copy.deepcopy(critic)
    with torch.no_grad():
        for net in (ap, cp):
            for p in net.parameters():
                p.add_(0.15 * p.abs().mean() * torch.randn(p.shape, device=DEV, generator=g))
        sp = std * torch.tensor([1.15, 0.9], device=DEV)
        obs = torch.randn(n, D, device=DEV, generator=g)
        mu = ap(obs)
        val = cp(obs).squeeze(-1) + 0.25 * torch.randn(n, device=DEV, generator=g)
        act = mu + sp * torch.randn(n, 2, device=DEV, generator=g)
        lp = torch.distributions.Normal(mu, sp).log_prob(act).sum(-1)
        ret = val + 0.5 * torch.randn(n, device=DEV, generator=g)
        adv = 0.3 + torch.randn(n, device=DEV, generator=g)
    slab = SimpleNamespace(obs_in=obs.contiguous(), actions=act.contiguous(), values=val.contiguous(), log_prob=lp.contiguous(),
                           mean=mu.contiguous())
    return slab, ret.contiguous(), adv.contiguous(), torch.randperm(n, device=DEV, generator=g)


def _synthetic(D, activation, R, n, seed):
    """One blob and R ranks' batches of n rows each."""
    from wheeledlab_b200.policy import pack_actor_critic
    actor, critic, std = _nets(D, activation, seed)
    blob = pack_actor_critic(actor, critic, std, D, DEV)
    g = torch.Generator(device=DEV).manual_seed(seed + 1)
    return blob, [_batch(actor, critic, std, D, n, g) for _ in range(R)]


def _replicas(blob, D, cfg, activation, R):
    from wheeledlab_b200.learner import FusedPPO, PPOExchange
    return [FusedPPO(blob.clone(), D, cfg, activation, exchange=ex) for ex in PPOExchange.local(R, D, DEV)]


def _bits(x):
    return x.contiguous().view(torch.int32)


# ---- R = 1 is the single-rank update -----------------------------------------------------------------------------------

@pytest.mark.parametrize("D,activation", [(14, "elu"), (5, "elu"), (689, "relu"), (3208, "relu")],
                         ids=["drift14", "narrow5", "elevation689", "visual3208"])
def test_one_rank_equals_the_single_rank_update(D, activation):
    _need_gpu()
    from wheeledlab_b200.learner import FusedPPO, PPOConfig, update_local_ranks
    cfg = PPOConfig()
    blob, [(slab, ret, adv, perm)] = _synthetic(D, activation, 1, 2048, seed=D)
    ref = FusedPPO(blob.clone(), D, cfg, activation)
    (dp,) = _replicas(blob, D, cfg, activation, 1)
    for k in range(2):                                    # whole updates, the second from the first's moments
        ref.update(slab, ret, adv, perm)
        update_local_ranks([dp], [(slab, ret, adv, perm)])
        torch.cuda.synchronize()
        for name, a, b in (("blob", ref.blob, dp.blob), ("m", ref.m, dp.m), ("v", ref.v, dp.v), ("state", ref.state, dp.state),
                           ("gradient", ref.last_gradient(), dp.last_gradient())):
            assert torch.equal(_bits(a), _bits(b)), f"update {k}: {name} differs from the single-rank update"
    assert not dp.exchange.failed()


# ---- R emulated ranks against a torch restatement of rsl_rl's multi-GPU update ------------------------------------------

def _forward_loss(r, cfg, o, a, v_old, lp_old, mu_old, s_old, R_, A):
    """rsl_rl's loss on one mini-batch (tests/ppo_reference.py's, per rank), with the rank's kl_mean."""
    mu = r.actor(o)
    sigma = r.std.expand_as(mu)
    dist = torch.distributions.Normal(mu, sigma, validate_args=False)
    lp = dist.log_prob(a).sum(dim=-1)
    value = r.critic(o).squeeze(-1)
    entropy = dist.entropy().sum(dim=-1)
    with torch.inference_mode():
        kl = torch.sum(torch.log(sigma / s_old + 1.0e-5) + (torch.square(s_old) + torch.square(mu_old - mu)) / (2.0 * torch.square(sigma)) - 0.5, dim=-1)
        kl_mean = torch.mean(kl)
    ratio = torch.exp(lp - lp_old)
    surrogate = torch.max(-A * ratio, -A * torch.clamp(ratio, 1.0 - cfg.clip_param, 1.0 + cfg.clip_param)).mean()
    if cfg.use_clipped_value_loss:
        value_clipped = v_old + (value - v_old).clamp(-cfg.clip_param, cfg.clip_param)
        value_loss = torch.max((value - R_).pow(2), (value_clipped - R_).pow(2)).mean()
    else:
        value_loss = (R_ - value).pow(2).mean()
    return surrogate + cfg.value_loss_coef * value_loss - cfg.entropy_coef * entropy.mean(), kl_mean


def torch_dp_update(blob, D, cfg, activation, batches, dtype):
    """rsl_rl's multi-GPU PPO.update() [UPSTREAM-RECALL] over R ranks, restated on TorchPPO: per mini-batch every rank
    back-propagates its own rows, the gradients are summed in rank order and divided by R (reduce_parameters), kl_mean is
    summed and divided by R before the adaptive rule, the rate is rounded to fp32 (rank 0 broadcasts it as a tensor), then
    clip_grad_norm_ and Adam.  Every replica then holds the same weights, so one model stands for all of them.
    Returns the model and the per-mini-batch trace (mean KL, rate, averaged gradient of the last mini-batch)."""
    from ppo_reference_relu import torch_ppo
    r = torch_ppo(blob, D, cfg, dtype, activation)
    R = len(batches)
    rows = []
    for slab, ret, adv, perm in batches:
        a = adv.reshape(-1).to(dtype)
        rows.append(dict(obs=slab.obs_in.reshape(-1, D).to(dtype), act=slab.actions.reshape(-1, 2).to(dtype),
                         v=slab.values.reshape(-1).to(dtype), lp=slab.log_prob.reshape(-1).to(dtype),
                         mu=slab.mean.reshape(-1, 2).to(dtype), ret=ret.reshape(-1).to(dtype),
                         adv=(a - a.mean()) / (a.std() + 1e-8), perm=perm))
    old_sigma = r.std.detach().clone()
    n = rows[0]["obs"].shape[0]
    B = n // cfg.num_mini_batches
    lr = cfg.learning_rate
    trace = []
    params = r.parameters()
    for _ in range(cfg.num_learning_epochs):
        for i in range(cfg.num_mini_batches):
            grads, kls = [], []
            for x in rows:
                idx = x["perm"][i * B:(i + 1) * B]
                for p in params:
                    p.grad = None
                loss, kl_mean = _forward_loss(r, cfg, x["obs"][idx], x["act"][idx], x["v"][idx], x["lp"][idx], x["mu"][idx],
                                              old_sigma.expand(B, 2), x["ret"][idx], x["adv"][idx])
                loss.backward()
                grads.append([p.grad.detach().clone() for p in params])
                kls.append(kl_mean)
            kl = kls[0].clone()
            for k in kls[1:]:
                kl = kl + k
            kl = kl / R
            if cfg.schedule == "adaptive":
                if kl > cfg.desired_kl * 2.0:
                    lr = max(1e-5, lr / 1.5)
                elif kl < cfg.desired_kl / 2.0 and kl > 0.0:
                    lr = min(1e-2, lr * 1.5)
                lr = torch.tensor(lr, dtype=torch.float32).item()
            for g in r.optimizer.param_groups:
                g["lr"] = lr
            for j, p in enumerate(params):
                s = grads[0][j].clone()
                for gr in grads[1:]:
                    s = s + gr[j]
                p.grad = s / R
            avg = r.grads()
            nn.utils.clip_grad_norm_(params, cfg.max_grad_norm)
            r.optimizer.step()
            trace.append({"kl": kl.item(), "lr": lr, "grads": avg})
    return r, trace


CASES = [  # (R, D, activation, cfg overrides)
    (2, 14, "elu", {}),
    (3, 14, "elu", {"use_clipped_value_loss": False, "max_grad_norm": 0.05}),
    (8, 14, "elu", {"schedule": "fixed"}),
    (2, 689, "relu", {}),
    (3, 37, "relu", {"schedule": "fixed", "max_grad_norm": 0.05}),
]


@pytest.mark.parametrize("R,D,activation,over", CASES,
                         ids=[f"R{c[0]}-{c[2]}{c[1]}-" + ("-".join(f"{k}={v}" for k, v in c[3].items()) or "default") for c in CASES])
def test_emulated_ranks_follow_the_torch_restatement(R, D, activation, over):
    _need_gpu()
    from wheeledlab_b200.learner import PPOConfig, update_local_ranks
    from wheeledlab_b200.policy import actor_critic_state_dict
    cfg = PPOConfig(num_learning_epochs=2, num_mini_batches=4, **over)
    blob, batches = _synthetic(D, activation, R, 8192, seed=7 * R + D)
    if activation == "relu":      # every ReLU unit and loss branch of the first mini-batch clear of its edge on every rank
        from test_ppo_wide_numerics_cpu import apply_margins
        apply_margins(blob, D, batches, 0, 8192, cfg)
    ref32, tr32 = torch_dp_update(blob.clone(), D, cfg, activation, batches, torch.float32)
    ref64, tr64 = torch_dp_update(blob.clone(), D, cfg, activation, batches, torch.float64)
    ppos = _replicas(blob, D, cfg, activation, R)
    update_local_ranks(ppos, batches)
    torch.cuda.synchronize()
    for q in ppos[1:]:
        for a, b in ((ppos[0].blob, q.blob), (ppos[0].m, q.m), (ppos[0].v, q.v), (ppos[0].history, q.history)):
            assert torch.equal(_bits(a), _bits(b)), "the replicas drifted apart"
    assert not any(q.exchange.failed() for q in ppos)
    # the trained networks, as tests/test_ppo_update_gpu.py judges a whole update: actor mean and critic value on every
    # rank's rows, fused and torch-fp32 weights both evaluated in fp64 against the fp64 run.  ELU only: on these synthetic
    # ReLU batches Adam amplifies the rounding of units at the ReLU edge over the trajectory -- the single-rank
    # wl_ppo_update_wide (which R = 1 reproduces bit for bit) and torch fp32 each drift 1e-3 from fp64 on some output, so
    # the ReLU cases are judged on the averaged gradient below, where fused and torch stand on the same weights.
    if activation == "elu":
        from ppo_reference_relu import torch_ppo
        from wheeledlab_b200.policy import load_actor_critic_state_dict
        obs = torch.cat([b[0].obs_in for b in batches])
        t32_blob = load_actor_critic_state_dict({k: v.float() for k, v in ref32.state_dict().items()}, D, device=DEV)
        fused_out = torch_ppo(ppos[0].blob, D, cfg, torch.float64, activation).forward(obs)
        t32_out = torch_ppo(t32_blob, D, cfg, torch.float64, activation).forward(obs)
        truth = ref64.forward(obs)
        for k, name in enumerate(("mean", "value")):
            ef, et = _err(fused_out[k], truth[k]), _err(t32_out[k], truth[k])
            assert ef <= max(4 * et, 1e-6), f"{name}: err {ef:.3g} vs torch fp32 {et:.3g}"
    # the averaged gradient per tensor, where fused and torch stand on the same weights: one update of one mini-batch
    one = PPOConfig(**{**cfg.__dict__, "num_learning_epochs": 1, "num_mini_batches": 1})
    g32, g64 = (torch_dp_update(blob.clone(), D, one, activation, batches, dt)[1][0]["grads"] for dt in (torch.float32, torch.float64))
    first = _replicas(blob, D, one, activation, R)
    update_local_ranks(first, batches)
    grad = actor_critic_state_dict(first[0].last_gradient(), D)
    for k in g64:
        ef, et = _err(grad[k], g64[k]), _err(g32[k], g64[k])
        assert ef <= max(4 * et, 1e-6), f"gradient {k}: err {ef:.3g} vs torch fp32 {et:.3g}"
    hist = ppos[0].history.cpu().double()
    assert torch.allclose(hist[:, 1], torch.tensor([t["lr"] for t in tr64], dtype=torch.float64), rtol=1e-6, atol=0)
    assert torch.allclose(hist[:, 0], torch.tensor([t["kl"] for t in tr64], dtype=torch.float64), rtol=1e-3, atol=1e-7)
    if cfg.schedule == "fixed":
        assert torch.all(hist[:, 1] == torch.tensor(cfg.learning_rate, dtype=torch.float32).double())


def _shard_rollouts(R, N, T, seed, blob, D):
    """R env shards (env_id_offset = r * N) rolled out from one blob, and the same R * N envs as one sim."""
    import wheeledlab_b200 as wl
    from wheeledlab_b200.policy import FusedPolicyRollout
    big = wl.WheeledSim(wl.drift_task(num_envs=R * N, seed=seed), DEV); big.startup(); big.reset(None, 0)
    whole = FusedPolicyRollout(big, blob.clone(), T).capture(0).run()
    sims = []
    for r in range(R):
        s = wl.WheeledSim(wl.drift_task(num_envs=N, seed=seed, env_id_offset=r * N), DEV); s.startup(); s.reset(None, 0)
        sims.append(s)
    return whole, sims


def test_lr_sequence_of_sharded_rollouts_equals_fp64_at_4096x128():
    """R = 2 ranks of 2048 envs x 128 steps (4096 x 128 in all), the reference Drift agent cfg: the 20 learning rates equal
    the fp64 restatement's, and the replicas stay bit-identical."""
    _need_gpu()
    from wheeledlab_b200.learner import PPOConfig, compute_returns, update_local_ranks
    from wheeledlab_b200.policy import FusedPolicyRollout, critic_value, pack_actor_critic
    R, N, T, D = 2, 2048, 128, 14
    cfg = PPOConfig()
    actor, critic, _ = _nets(D, "elu", 3)
    blob = pack_actor_critic(actor, critic, torch.ones(2, device=DEV), D, DEV)
    _, sims = _shard_rollouts(R, N, T, 5, blob, D)
    g = torch.Generator(device=DEV).manual_seed(3)
    batches = []
    for s in sims:
        roll = FusedPolicyRollout(s, blob.clone(), T).capture(0)
        slab = roll.run()
        last = critic_value(blob, D, roll.obs0)
        ret, adv = compute_returns(slab.rewards, slab.values, last, slab.terminated | slab.truncated, cfg.gamma, cfg.lam,
                                   time_outs=slab.truncated)
        batches.append((slab, ret, adv, torch.randperm(T * N, device=DEV, generator=g)))
    _, tr64 = torch_dp_update(blob.clone(), D, cfg, "elu", batches, torch.float64)
    for t in tr64:                                        # the seed keeps every KL clear of the schedule's thresholds
        for thr in (2 * cfg.desired_kl, cfg.desired_kl / 2):
            assert abs(t["kl"] - thr) > 1e-3 * thr, f"KL {t['kl']} within 1e-3 of {thr}: pick another seed"
    ppos = _replicas(blob, D, cfg, "elu", R)
    update_local_ranks(ppos, batches)
    hist = ppos[0].history.cpu().double()
    lrs = torch.tensor([t["lr"] for t in tr64], dtype=torch.float64)
    assert hist.shape[0] == 20 and torch.equal(hist[:, 1], lrs), (hist[:, 1], lrs)
    assert len(set(lrs.tolist())) > 1, "the lr never moved"
    for q in ppos[1:]:
        assert torch.equal(_bits(ppos[0].blob), _bits(q.blob)) and torch.equal(_bits(ppos[0].v), _bits(q.v))


# ---- sharded iterations and the captured one-process iteration ----------------------------------------------------------

def _local_iterations(R, N, T, seed, blob, capture):
    import wheeledlab_b200 as wl
    from wheeledlab_b200.learner import LocalRanksIteration, PPOConfig, PPOExchange, PPOIteration
    its = []
    for r, ex in enumerate(PPOExchange.local(R, 14, DEV)):
        s = wl.WheeledSim(wl.drift_task(num_envs=N, seed=seed, env_id_offset=r * N), DEV); s.startup(); s.reset(None, 0)
        its.append(PPOIteration(s, blob.clone(), PPOConfig(), T, episode_stats=True, exchange=ex))
    return LocalRanksIteration(its).start(0, capture=capture)


SLAB = ("obs_in", "actions", "values", "log_prob", "mean", "rewards", "terminated", "truncated")


def test_env_shards_concatenate_to_one_rollout_and_replicas_stay_equal():
    _need_gpu()
    from wheeledlab_b200.policy import pack_actor_critic
    R, N, T = 3, 512, 16
    actor, critic, std = _nets(14, "elu", 9, std=(1.0, 1.0))
    blob = pack_actor_critic(actor, critic, std, 14, DEV)
    whole, _ = _shard_rollouts(R, N, T, 4, blob, 14)
    group = _local_iterations(R, N, T, 4, blob, capture=False)
    g = torch.Generator(device=DEV).manual_seed(2)
    for k in range(3):
        group.run([torch.randperm(N * T, device=DEV, generator=g) for _ in range(R)])
        torch.cuda.synchronize()
        if k == 0:
            for f in SLAB:
                cat = torch.cat([getattr(it.roll.slab, f) for it in group.its], dim=1)
                assert torch.equal(cat.view(torch.uint8), getattr(whole, f).view(torch.uint8)), f"slab field {f}"
        a = group.its[0]
        for b in group.its[1:]:
            for x, y in ((a.blob, b.blob), (a.ppo.m, b.ppo.m), (a.ppo.v, b.ppo.v)):
                assert torch.equal(_bits(x), _bits(y)), f"iteration {k}: replicas differ"
            assert torch.equal(_bits(a.ppo.history), _bits(b.ppo.history))


def test_captured_one_process_iteration_replays_as_the_eager_sequence():
    _need_gpu()
    from wheeledlab_b200.policy import pack_actor_critic
    R, N, T = 2, 1024, 32
    actor, critic, std = _nets(14, "elu", 9, std=(1.0, 1.0))
    blob = pack_actor_critic(actor, critic, std, 14, DEV)
    eager = _local_iterations(R, N, T, 4, blob, capture=False)
    graph = _local_iterations(R, N, T, 4, blob, capture=True)
    g = torch.Generator(device=DEV).manual_seed(1)
    for k in range(4):
        perms = [torch.randperm(N * T, device=DEV, generator=g) for _ in range(R)]
        eager.run(perms)
        graph.run(perms)
        torch.cuda.synchronize()
        for a, b in zip(eager.its, graph.its):
            for name, x, y in (("blob", a.blob, b.blob), ("m", a.ppo.m, b.ppo.m), ("v", a.ppo.v, b.ppo.v),
                               ("state", a.ppo.state, b.ppo.state), ("slab", a.roll.slab.flat, b.roll.slab.flat),
                               ("episodes", a.episodes.state, b.episodes.state), ("summary", a.summary, b.summary)):
                assert torch.equal(x.view(torch.uint8), y.view(torch.uint8)), f"replay {k}: {name}"
        for ex_a, ex_b in zip(eager.its, graph.its):     # the device epoch advanced by the same rounds
            assert torch.equal(ex_a.ppo.exchange.buffer[:8], ex_b.ppo.exchange.buffer[:8])
    epoch = int(graph.its[0].ppo.exchange.buffer[:4].view(torch.int32).item())
    assert epoch == 4 * 20 and not graph.its[0].ppo.exchange.failed()


def test_local_buffers_on_different_devices_are_refused():
    _need_gpu()
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    import ctypes as C
    import wheeledlab_b200 as wl
    from wheeledlab_b200.learner import PPOConfig, PPOExchange
    blob, [(slab, ret, adv, perm)] = _synthetic(14, "elu", 1, 1024, seed=1)
    nb = PPOExchange.nbytes(14)
    bufs = [torch.zeros(nb, dtype=torch.uint8, device=f"cuda:{d}") for d in (0, 1)]
    ppos = _replicas(blob, 14, PPOConfig(), "elu", 2)
    for q in ppos:
        q.exchange.ptrs = (C.c_void_p * 2)(*[b.data_ptr() for b in bufs])
    from wheeledlab_b200.learner import update_local_ranks
    with pytest.raises(wl.WlError, match="different devices"):
        update_local_ranks(ppos, [(slab, ret, adv, perm)] * 2)


def test_two_process_data_parallel_update_and_runner(tmp_path):
    """tools/ppo_dp_check.py under torchrun on 2 GPUs: replicas bit-identical over peer memory, equal to the one-process
    form, and the runner trains and resumes from rank 0's checkpoint (skipped on a single-GPU machine)."""
    _need_gpu()
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import subprocess
    import sys
    from pathlib import Path
    root = Path(__file__).resolve().parent.parent
    out = tmp_path / "ok.txt"
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", "29741", str(root / "tools" / "ppo_dp_check.py"), "--out", str(out)]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0 and out.read_text().startswith("ok"), r.stderr[-2000:]
