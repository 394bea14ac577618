"""Training an env that has device terms: FusedOnPolicyRunner's iteration with T x (policy_act, wl_step_terms) captured in
the one graph, its Episode_* keys, checkpoints that resume, and the one-process data-parallel iteration."""
import pytest
import torch

pytestmark = pytest.mark.gpu

if not torch.cuda.is_available():
    pytest.skip("needs a CUDA device", allow_module_level=True)

import wheeledlab_b200 as wl                                   # noqa: E402
from wheeledlab_b200 import device_terms as dtm                # noqa: E402
from wheeledlab_b200.env import ManagerBasedRLEnv              # noqa: E402

DEV = "cuda:0"
T = 8


def _env(kind, n, offset=0):
    spec = wl.elevation_task(num_envs=n, seed=4, env_id_offset=offset) if kind == "elevation" else \
        wl.drift_task(num_envs=n, seed=4, env_id_offset=offset)
    env = ManagerBasedRLEnv(spec, device=DEV)
    env.add_device_reward_term("steep", dtm.resolve("steep_penalty", dtm.ELEVATION), -1.0, {"thresh_pitch": 0.05})
    env.add_device_reward_term("up", dtm.resolve("upright_penalty", dtm.ELEVATION), -0.01, {"thresh_deg": 2.0})
    env.add_device_termination_term("flip", dtm.resolve("roll_over", dtm.VISUAL))
    return env


def _runner(env, activation, **kw):
    from wheeledlab_b200.learner import FusedOnPolicyRunner
    from wheeledlab_b200.runs import agent_cfg
    torch.manual_seed(0)                                    # the same initial weights for every runner
    return FusedOnPolicyRunner(env, agent_cfg(activation, steps=T, save_interval=1), device=DEV, **kw)


def _bits(x):
    return x.contiguous().view(torch.uint8)


def test_runner_iteration_is_one_graph_with_the_device_terms_and_logs_their_means():
    env = _env("elevation", 256)
    r = _runner(env, "relu")
    torch.manual_seed(3)
    rows = []
    r.callback = lambda k, log: rows.append(r.it.roll.term_logs.clone())
    log = r.learn(2)
    assert r.it.graph is not None and r.it.roll.device_terms
    assert env.common_step_counter == 2 * T
    means = r.it.roll.term_logs[:, :3].cpu().double().mean(0).tolist()
    for name, want in zip(["Episode_Reward/steep", "Episode_Reward/up", "Episode_Termination/flip"], means):
        assert log[name] == want, name


def test_captured_device_term_iteration_equals_the_eager_one():
    from wheeledlab_b200.learner import PPOConfig, device_terms_iteration
    from wheeledlab_b200.policy import pack_actor_critic
    n, D = 256, 689
    mk = lambda out: torch.nn.Sequential(torch.nn.Linear(D, 64), torch.nn.ReLU(), torch.nn.Linear(64, 64), torch.nn.ReLU(), torch.nn.Linear(64, out))
    torch.manual_seed(5)
    blob = pack_actor_critic(mk(2), mk(1), torch.full((2,), 1.0), D, DEV)
    ea, eb = _env("elevation", n), _env("elevation", n)
    for e in (ea, eb):
        e.reset()
    a = device_terms_iteration(ea, blob.clone(), PPOConfig(), T, "relu").start(0, capture=False)
    b = device_terms_iteration(eb, blob.clone(), PPOConfig(), T, "relu").start(0, capture=True)
    g = torch.Generator(device=DEV).manual_seed(2)
    for k in range(3):
        perm = torch.randperm(n * T, device=DEV, generator=g)
        a.run(perm); b.run(perm)
        torch.cuda.synchronize()
        for name, x, y in (("blob", a.blob, b.blob), ("m", a.ppo.m, b.ppo.m), ("slab", a.roll.slab.flat, b.roll.slab.flat),
                           ("term_logs", a.roll.term_logs, b.roll.term_logs), ("episodes", a.episodes.state, b.episodes.state)):
            assert torch.equal(_bits(x), _bits(y)), f"iteration {k}: {name}"
        assert torch.equal(ea.sim.groups, eb.sim.groups)


def test_device_terms_change_the_rollout_rewards():
    """The same weights and counters without the device terms give different rewards (the terms are in the rollout)."""
    from wheeledlab_b200.learner import PPOConfig, PPOIteration, device_terms_iteration
    from wheeledlab_b200.policy import pack_actor_critic
    n, D = 256, 14
    mk = lambda out: torch.nn.Sequential(torch.nn.Linear(D, 64), torch.nn.ELU(), torch.nn.Linear(64, 64), torch.nn.ELU(), torch.nn.Linear(64, out))
    torch.manual_seed(6)
    blob = pack_actor_critic(mk(2), mk(1), torch.full((2,), 1.0), D, DEV)
    e = ManagerBasedRLEnv(wl.drift_task(num_envs=n, seed=4), device=DEV)
    e.add_device_reward_term("fv", dtm.resolve("forward_vel", dtm.ELEVATION), 3.0)
    p = ManagerBasedRLEnv(wl.drift_task(num_envs=n, seed=4), device=DEV)
    for x in (e, p):
        x.reset()
    a = device_terms_iteration(e, blob.clone(), PPOConfig(), T, "elu").start(0)
    b = PPOIteration(p.sim, blob.clone(), PPOConfig(), T, "elu", episode_stats=True).start(0)
    perm = torch.randperm(n * T, device=DEV)
    a.run(perm); b.run(perm)
    torch.cuda.synchronize()
    assert torch.equal(a.roll.slab.actions[0], b.roll.slab.actions[0])
    assert not torch.equal(a.roll.slab.rewards[0], b.roll.slab.rewards[0])


def test_checkpoint_resumes_bit_for_bit(tmp_path):
    from wheeledlab_b200.learner import FusedOnPolicyRunner
    from wheeledlab_b200.runs import agent_cfg
    env_a, env_b = _env("drift", 256), _env("drift", 256)
    a, b = _runner(env_a, "elu", log_dir=str(tmp_path)), _runner(env_b, "elu")
    for r in (a, b):
        torch.manual_seed(21)
        r.learn(2)
    c = FusedOnPolicyRunner(env_b, agent_cfg("elu", steps=T, save_interval=1), device=DEV)
    c.load(str(tmp_path / "models" / "model_1.pt"))
    assert c.current_learning_iteration == 1
    a.alg.state[0] = c.alg.cfg.learning_rate
    for r in (a, c):
        torch.manual_seed(22)
        r.learn(1)
    torch.cuda.synchronize()
    assert env_a.common_step_counter == env_b.common_step_counter == 3 * T
    for name, x, y in (("blob", a.blob, c.blob), ("m", a.alg.m, c.alg.m), ("v", a.alg.v, c.alg.v)):
        assert torch.equal(_bits(x), _bits(y)), name


def test_one_process_data_parallel_iteration_keeps_replicas_equal():
    from wheeledlab_b200.learner import LocalRanksIteration, PPOConfig, PPOExchange, device_terms_iteration
    from wheeledlab_b200.policy import pack_actor_critic
    R, n, D = 2, 512, 14
    mk = lambda out: torch.nn.Sequential(torch.nn.Linear(D, 64), torch.nn.ELU(), torch.nn.Linear(64, 64), torch.nn.ELU(), torch.nn.Linear(64, out))
    torch.manual_seed(7)
    blob = pack_actor_critic(mk(2), mk(1), torch.full((2,), 1.0), D, DEV)
    its = []
    for r, ex in enumerate(PPOExchange.local(R, D, DEV)):
        e = _env("drift", n, offset=r * n); e.reset()
        its.append(device_terms_iteration(e, blob.clone(), PPOConfig(), T, "elu", exchange=ex))
    group = LocalRanksIteration(its).start(0, capture=True)
    g = torch.Generator(device=DEV).manual_seed(1)
    for k in range(3):
        group.run([torch.randperm(n * T, device=DEV, generator=g) for _ in range(R)])
        torch.cuda.synchronize()
        a, b = group.its
        for x, y in ((a.blob, b.blob), (a.ppo.m, b.ppo.m), (a.ppo.v, b.ppo.v)):
            assert torch.equal(_bits(x), _bits(y)), f"iteration {k}: replicas differ"
        assert not torch.equal(a.roll.slab.rewards, b.roll.slab.rewards)      # different env shards
    assert not group.its[0].ppo.exchange.failed()
