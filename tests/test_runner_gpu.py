"""The runner on the device: wl_episode_stats (learner.EpisodeStatistics) against the reference runner's bookkeeping restated
literally (a deque(maxlen=100), fp32 torch += per step, nonzero() order), on synthetic slabs and on the slabs real runs
produce, under graph replay; FusedOnPolicyRunner's checkpoints resumed bit for bit; checkpoints exchanged with the torch
restatement of rsl_rl's PPO (tests/ppo_reference.py)."""
import math
import statistics
from collections import deque

import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")


class RunnerBookkeeping:
    """modified_rsl_rl_runner.py:55-63, :99-109, literally."""

    def __init__(self, n):
        self.rewbuffer, self.lenbuffer = deque(maxlen=100), deque(maxlen=100)
        self.cur_reward_sum = torch.zeros(n, dtype=torch.float, device=DEV)
        self.cur_episode_length = torch.zeros(n, dtype=torch.float, device=DEV)

    def step(self, rewards, dones):
        self.cur_reward_sum += rewards
        self.cur_episode_length += 1
        new_ids = (dones > 0).nonzero(as_tuple=False)
        self.rewbuffer.extend(self.cur_reward_sum[new_ids][:, 0].cpu().numpy().tolist())
        self.lenbuffer.extend(self.cur_episode_length[new_ids][:, 0].cpu().numpy().tolist())
        self.cur_reward_sum[new_ids] = 0
        self.cur_episode_length[new_ids] = 0

    def rollout(self, rewards, terminated, truncated):
        for t in range(rewards.shape[0]):
            self.step(rewards[t], terminated[t] | truncated[t])


def _assert_same(ep, ref, what):
    """ring contents, fill, carries bit-identical; the means equal statistics.mean to fp64 rounding."""
    rets, lens = ep.ring()
    assert rets == list(ref.rewbuffer), f"{what}: ring returns"
    assert lens == list(ref.lenbuffer), f"{what}: ring lengths"
    assert torch.equal(ep.cur_return.view(torch.int32), ref.cur_reward_sum.view(torch.int32)), f"{what}: running returns"
    assert torch.equal(ep.cur_length.view(torch.int32), ref.cur_episode_length.view(torch.int32)), f"{what}: running lengths"
    fill, _, _ = ep.counts.tolist()
    mean_ret, mean_len = ep.means.tolist()
    assert fill == len(ref.rewbuffer), what
    if fill == 0:
        assert (mean_ret, mean_len) == (0.0, 0.0), what
        return
    for got, want in ((mean_ret, statistics.mean(ref.rewbuffer)), (mean_len, statistics.mean(ref.lenbuffer))):
        assert abs(got - want) <= 4 * math.ulp(want), f"{what}: mean {got!r} vs statistics.mean {want!r}"


def _slab(T, N, case, it, g):
    """rewards with magnitudes over six decades (fp32 order matters) and the done pattern of `case`."""
    rew = (torch.randn(T, N, device=DEV, generator=g) * 10.0 ** torch.randint(-3, 3, (T, N), device=DEV, generator=g)).float()
    term = torch.zeros(T, N, dtype=torch.uint8, device=DEV)
    trunc = torch.zeros(T, N, dtype=torch.uint8, device=DEV)
    u = lambda p: (torch.rand(T, N, device=DEV, generator=g) < p).to(torch.uint8)
    if case == "random":
        term, trunc = u(0.02), u(0.01)
    elif case == "sparse":                                  # episodes span iteration boundaries
        term = u(0.3 / (T * N) ** 0.5)
    elif case == "exactly_100":
        idx = torch.randperm(T * N, device=DEV, generator=g)[:100]
        term.view(-1)[idx] = 1
    elif case == "burst":                                   # every env ends at one t (more than 100 at once), a few others
        term, trunc = u(0.005), u(0.005)
        trunc[min(T - 1, 3 + it)] = 1
    elif case == "t0":
        term[0] = u(0.5)[0]
        trunc = u(0.01)
    elif case == "both":                                    # terminated and truncated on the same step
        term = u(0.03)
        trunc = term.clone()
        trunc |= u(0.01)
    elif case != "none":
        raise ValueError(case)
    return rew.contiguous(), term.contiguous(), trunc.contiguous()


CASES = [(1, 1, "random"), (1, 33, "random"), (1, 4096, "random"), (128, 1, "random"), (128, 33, "random"), (128, 4096, "random"),
         (128, 33, "none"), (128, 4096, "exactly_100"), (128, 4096, "burst"), (1, 4096, "burst"), (128, 33, "sparse"),
         (128, 4096, "sparse"), (128, 4096, "t0"), (128, 33, "both"), (128, 4096, "both"), (7, 1000, "random"),
         # T > 1024 runs the ring kernel's 1024-step loop more than once (4096 = WL_EP_MAX_T); N = 1057 has 34 done words
         # per row, neither a multiple of 32 nor one chunk
         (17, 1057, "random"), (1025, 1057, "random"), (4096, 33, "random"), (4096, 1057, "both"), (128, 1057, "burst")]


@pytest.mark.parametrize("T,N,case", CASES)
def test_episode_stats_match_the_runner_bookkeeping(T, N, case):
    _need_gpu()
    from wheeledlab_b200.learner import EpisodeStatistics
    g = torch.Generator(device=DEV).manual_seed(T * 7919 + N)
    ep, ref = EpisodeStatistics(N, T, DEV), RunnerBookkeeping(N)
    iters = 40 if T == 1 else 4
    for it in range(iters):
        rew, term, trunc = _slab(T, N, case, it, g)
        ep.update(rew, term, trunc)
        ref.rollout(rew, term, trunc)
        assert ep.counts[2].item() == int((term | trunc).sum()), "finished this iteration"
        _assert_same(ep, ref, f"{case} T={T} N={N} iteration {it}")
    if case == "none":
        assert ep.counts[0].item() == 0
    if case == "exactly_100":
        assert len(ref.rewbuffer) == 100
    ep.reset()
    assert ep.counts.tolist() == [0, 0, 0] and not ep.cur_return.any() and not ep.cur_length.any()


def test_episode_stats_graph_replay_equals_the_eager_sequence():
    _need_gpu()
    from wheeledlab_b200.learner import EpisodeStatistics
    T, N = 128, 4096
    g = torch.Generator(device=DEV).manual_seed(5)
    bufs = [torch.zeros(T, N, device=DEV), torch.zeros(T, N, dtype=torch.uint8, device=DEV), torch.zeros(T, N, dtype=torch.uint8, device=DEV)]
    eager, graphed = EpisodeStatistics(N, T, DEV), EpisodeStatistics(N, T, DEV)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s), torch.cuda.graph(graph, stream=s):
        graphed.update(*bufs)
    torch.cuda.current_stream().wait_stream(s)
    graphed.reset()                                         # (capture does not run the kernels, but start from zero anyway)
    for it in range(6):
        for b, x in zip(bufs, _slab(T, N, "random" if it % 2 else "burst", it, g)):
            b.copy_(x)
        graph.replay()
        eager.update(*bufs)
        torch.cuda.synchronize()
        assert torch.equal(graphed.state, eager.state), f"iteration {it}: state"
        assert torch.equal(graphed.cur_return.view(torch.int32), eager.cur_return.view(torch.int32))
        assert torch.equal(graphed.cur_length.view(torch.int32), eager.cur_length.view(torch.int32))


def _agent_cfg(activation, save_interval=50, **alg):
    from dataclasses import asdict
    from wheeledlab_b200.learner import PPOConfig
    return {"num_steps_per_env": 128, "save_interval": save_interval, "empirical_normalization": False,
            "policy": {"class_name": "ActorCritic", "init_noise_std": 1.0, "actor_hidden_dims": [64, 64], "critic_hidden_dims": [64, 64],
                       "activation": activation},
            "algorithm": {"class_name": "PPO", **asdict(PPOConfig(**alg))}}


@pytest.mark.parametrize("task,n,activation", [("Isaac-MushrDriftRL-v0", 4096, "elu"), ("Isaac-MushrElevationRL-v0", 1024, "relu")])
def test_runner_statistics_on_real_rollouts(task, n, activation):
    _need_gpu()
    import wheeledlab_b200 as wl
    from wheeledlab_b200.learner import FusedOnPolicyRunner, PPOIteration
    torch.manual_seed(0)
    env = wl.make(task, device=DEV, num_envs=n, seed=3)
    runner = FusedOnPolicyRunner(env, _agent_cfg(activation), device=DEV)
    ref = RunnerBookkeeping(n)
    seen = []

    def check(it, log):
        slab = runner.it.roll.slab
        ref.rollout(slab.rewards, slab.terminated, slab.truncated)
        _assert_same(runner.it.episodes, ref, f"{task} iteration {it}")
        if ref.rewbuffer:
            assert log["Train/mean_reward"] == runner.it.episodes.means[0].item()
            assert abs(log["Train/mean_episode_length"] - statistics.mean(ref.lenbuffer)) <= 4 * math.ulp(statistics.mean(ref.lenbuffer))
        else:
            assert "Train/mean_reward" not in log and "Train/mean_episode_length" not in log
        assert set(PPOIteration.SUMMARY) <= set(log) and set(env._log_index) <= set(log) and log["Perf/total_fps"] > 0
        want_lr = runner.alg.state[0].item()
        assert log["Loss/learning_rate"] == want_lr
        logs = runner.it.roll.logs.double().mean(0)
        for name, col in env._log_index.items():
            assert log[name] == pytest.approx(logs[col].item(), rel=1e-12, abs=1e-30), name
        seen.append(it)

    runner.callback = check
    runner.learn(3)
    assert seen == [0, 1, 2] and env.common_step_counter == 3 * 128 and runner.current_learning_iteration == 2


def test_resume_continues_bit_for_bit(tmp_path):
    _need_gpu()
    import wheeledlab_b200 as wl
    from wheeledlab_b200.learner import FusedOnPolicyRunner
    torch.manual_seed(1)
    env = wl.make("Isaac-MushrDriftRL-v0", device=DEV, num_envs=1024, seed=4)
    cfg = _agent_cfg("elu", save_interval=1)
    a = FusedOnPolicyRunner(env, cfg, log_dir=str(tmp_path), device=DEV)
    a.learn(2)                                                            # iterations 0, 1 -> models/model_0.pt, model_1.pt
    ck = torch.load(tmp_path / "models" / "model_1.pt")
    assert set(ck) == {"model_state_dict", "optimizer_state_dict", "iter", "infos"} and ck["iter"] == 1
    saved_lr = ck["optimizer_state_dict"]["param_groups"][0]["lr"]
    b = FusedOnPolicyRunner(env, cfg, device=DEV)
    assert b.load(str(tmp_path / "models" / "model_1.pt")) is None and b.current_learning_iteration == 1
    assert torch.equal(b.blob.view(torch.int32), a.blob.view(torch.int32))
    assert torch.equal(b.alg.m.view(torch.int32), a.alg.m.view(torch.int32)) and torch.equal(b.alg.v.view(torch.int32), a.alg.v.view(torch.int32))
    assert b.alg.state[1].item() == a.alg.state[1].item() == 2 * 20                   # 5 epochs x 4 mini-batches per update
    assert b.alg.state[0].item() == pytest.approx(1e-3) and saved_lr == a.alg.state[0].item()    # lr after a load: the cfg's
    # A's next iteration from the same learning rate B starts from; then B's update on A's slab and permutation
    a.alg.state[0] = cfg["algorithm"]["learning_rate"]
    a.learn(1)                                                            # iteration 2
    b.it.roll.slab, b.it.roll.obs0 = a.it.roll.slab, a.it.roll.obs0
    b.it.perm.copy_(a.it.perm)
    b.it._learn()
    torch.cuda.synchronize()
    for name, x, y in (("blob", a.blob, b.blob), ("m", a.alg.m, b.alg.m), ("v", a.alg.v, b.alg.v)):
        assert torch.equal(x.view(torch.int32), y.view(torch.int32)), name
    assert a.alg.state[:2].tolist() == b.alg.state[:2].tolist()
    assert torch.equal(a.alg.history, b.alg.history)
    # a malformed checkpoint is refused before anything changes
    bad = dict(ck, model_state_dict={k: v for k, v in ck["model_state_dict"].items() if k != "critic.4.bias"})
    torch.save(bad, tmp_path / "bad.pt")
    before = b.blob.clone()
    with pytest.raises(ValueError):
        b.load(str(tmp_path / "bad.pt"))
    torch.save({"model_state_dict": ck["model_state_dict"]}, tmp_path / "no_iter.pt")
    with pytest.raises(ValueError):
        b.load(str(tmp_path / "no_iter.pt"))
    assert torch.equal(before, b.blob)


def _err(x, ref):
    return ((x.double() - ref.double()).norm() / ref.double().norm()).item()


def _batch(blob, D, n, seed):
    """A batch collected by a perturbed copy of the network (both clip branches are taken)."""
    from types import SimpleNamespace
    from ppo_reference import TorchPPO
    from wheeledlab_b200.learner import PPOConfig
    g = torch.Generator(device=DEV).manual_seed(seed)
    ref = TorchPPO(blob, D, PPOConfig())
    with torch.no_grad():
        for p in ref.parameters():
            p.add_(0.15 * p.abs().mean() * torch.randn(p.shape, device=DEV, generator=g))
        obs = torch.randn(n, D, device=DEV, generator=g)
        mu, val = ref.forward(obs)
        sp = ref.std.detach()
        act = mu + sp * torch.randn(n, 2, device=DEV, generator=g)
        lp = torch.distributions.Normal(mu, sp).log_prob(act).sum(-1)
        ret = val + 0.5 * torch.randn(n, device=DEV, generator=g)
        adv = 0.3 + torch.randn(n, device=DEV, generator=g)
    slab = SimpleNamespace(obs_in=obs.contiguous(), actions=act.contiguous(), values=val.contiguous(), log_prob=lp.contiguous(),
                           mean=mu.contiguous())
    return slab, ret.contiguous(), adv.contiguous(), torch.randperm(n, device=DEV, generator=g)


def _torch_update(r, batch):
    slab, ret, adv, perm = batch
    return r.update(slab.obs_in, slab.actions, slab.values, slab.log_prob, slab.mean, ret, adv, perm)


def test_checkpoints_exchange_with_torch_ppo(tmp_path):
    _need_gpu()
    from ppo_reference import TorchPPO
    from wheeledlab_b200.learner import FusedPPO, PPOConfig
    from wheeledlab_b200.policy import actor_critic_state_dict, load_actor_critic_state_dict, pack_actor_critic
    D, n = 14, 16384
    cfg = PPOConfig(num_learning_epochs=2)
    torch.manual_seed(2)
    mk = lambda out: torch.nn.Sequential(torch.nn.Linear(D, 64), torch.nn.ELU(), torch.nn.Linear(64, 64), torch.nn.ELU(), torch.nn.Linear(64, out))
    blob0 = pack_actor_critic(mk(2), mk(1), torch.tensor([0.9, 1.1]), D, DEV)
    # torch (fp32) trains a few updates; its checkpoint loads into the fused learner exactly
    t32 = TorchPPO(blob0, D, cfg)
    for s in range(2):
        _torch_update(t32, _batch(blob0, D, n, 10 + s))
    torch.save({"model_state_dict": t32.state_dict(), "optimizer_state_dict": t32.optimizer.state_dict(), "iter": 7, "infos": None},
               tmp_path / "torch.pt")
    ck = torch.load(tmp_path / "torch.pt")
    blob = load_actor_critic_state_dict(ck["model_state_dict"], D, device=DEV)
    fused = FusedPPO(blob, D, cfg)
    fused.load_optimizer_state_dict(ck["optimizer_state_dict"])
    for i, p in enumerate(t32.parameters()):
        st = t32.optimizer.state[p]
        name = list(actor_critic_state_dict(blob, D))[i]
        for mine, theirs in ((actor_critic_state_dict(fused.m, D)[name], st["exp_avg"]), (actor_critic_state_dict(fused.v, D)[name], st["exp_avg_sq"])):
            assert torch.equal(mine.view(torch.int32), theirs.view(torch.int32)), name
        assert torch.equal(actor_critic_state_dict(blob, D)[name], p.detach()), name
    assert fused.state[1].item() == float(t32.optimizer.state[t32.parameters()[0]]["step"])
    # the next update of each, from the same checkpoint (torch's adaptive rate also restarts from the cfg's), against fp64
    batch = _batch(blob, D, n, 20)
    refs = {}
    for dt in (torch.float32, torch.float64):
        r = TorchPPO(blob, D, cfg, dt)
        r.optimizer.load_state_dict(ck["optimizer_state_dict"])
        _torch_update(r, batch)
        refs[dt] = r
    fused.update(*batch)
    obs = batch[0].obs_in[:4096]
    truth = refs[torch.float64].forward(obs)
    f64 = TorchPPO(blob, D, cfg, torch.float64).forward(obs)
    t = TorchPPO(load_actor_critic_state_dict({k: v.float() for k, v in refs[torch.float32].state_dict().items()}, D, device=DEV),
                 D, cfg, torch.float64).forward(obs)
    for k, name in enumerate(("mean", "value")):
        ef, et = _err(f64[k], truth[k]), _err(t[k], truth[k])
        assert ef <= max(4 * et, 1e-6), f"{name}: fused err {ef:.3g} vs torch fp32 {et:.3g}"
    # a fused checkpoint loads into torch's ActorCritic + Adam, and the next updates agree the same way
    sd = {"model_state_dict": actor_critic_state_dict(blob, D), "optimizer_state_dict": fused.optimizer_state_dict()}
    torch.save(sd, tmp_path / "fused.pt")
    sd = torch.load(tmp_path / "fused.pt")
    back = TorchPPO(load_actor_critic_state_dict(sd["model_state_dict"], D, device=DEV), D, cfg)
    back.optimizer.load_state_dict(sd["optimizer_state_dict"])
    for i, p in enumerate(back.parameters()):
        name = list(sd["model_state_dict"])[i]
        assert torch.equal(p.detach(), sd["model_state_dict"][name])
        assert torch.equal(back.optimizer.state[p]["exp_avg"], sd["optimizer_state_dict"]["state"][i]["exp_avg"])
    batch = _batch(blob, D, n, 30)
    r64 = TorchPPO(blob, D, cfg, torch.float64)
    r64.optimizer.load_state_dict(sd["optimizer_state_dict"])
    _torch_update(r64, batch)
    _torch_update(back, batch)
    fused.load_optimizer_state_dict(sd["optimizer_state_dict"])        # (same lr-after-load start as the torch learners)
    fused.update(*batch)
    truth = r64.forward(obs)
    f64 = TorchPPO(blob, D, cfg, torch.float64).forward(obs)
    t = TorchPPO(load_actor_critic_state_dict({k: v.float() for k, v in back.state_dict().items()}, D, device=DEV), D, cfg,
                 torch.float64).forward(obs)
    for k, name in enumerate(("mean", "value")):
        ef, et = _err(f64[k], truth[k]), _err(t[k], truth[k])
        assert ef <= max(4 * et, 1e-6), f"{name} after the fused checkpoint: fused err {ef:.3g} vs torch fp32 {et:.3g}"
