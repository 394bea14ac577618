"""The Elevation asymmetric actor-critic on the device (DESIGN 6s):
- the row critic (wl_set_row_critic, wl_critic_observe): its first 689 columns equal the CPU twin with no noise and the
  critic's clips and scales, and the policy row of a noise-free handle, bit for bit; its extra columns equal the state views;
  at N = 1, 33 (N * Dc odd) and 4096, on both scans, on host and device counters, across resets; a handle with Gaussian noise
  on every column has the critic row of the noise-free one;
- wl_policy_act_wide_asym: actions, mean and log-prob are wl_policy_act's bit for bit, the value too on the policy row, and
  against fp64 otherwise -- with the critic's chunks fewer than, as many as and more than the actor's;
- wl_ppo_update_wide_asym: on the policy row it is wl_ppo_update_wide bit for bit; its gradient meets the 4x torch-fp32 bar
  against fp64 at several Dc; padding is never stepped; runs and graph replays are reproducible;
- the iteration and the runner: one graph that equals the eager sequence, the symmetric iteration on the policy row, and a
  noisy-row-terms Elevation env with a row critic that trains, saves, loads, resumes and plays."""
import copy
import sys
from pathlib import Path
from types import SimpleNamespace

import numpy as np
import pytest
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "tests"))

pytestmark = pytest.mark.gpu

if not torch.cuda.is_available():
    pytest.skip("needs a CUDA device", allow_module_level=True)

import wheeledlab_b200 as wl                                   # noqa: E402
import row_terms_oracle as R                                   # noqa: E402
from wheeledlab_b200._lib import WlError                       # noqa: E402
from wheeledlab_b200.sim import WheeledSim                     # noqa: E402

DEV = "cuda:0"
D = 689
POLICY_GAUSS = [                                               # Gaussian noise on every column
    ("goal_relative_xyz", ("gaussian", 0.25, 0.5), (-3.0, 7.0), (2.0, -0.5)),
    ("root_euler_xyz", ("gaussian", -0.2, 0.6), None, 1.5),
    ("base_lin_vel", ("gaussian", -0.1, 0.3), (-4.0, 2.5), None),
    ("base_ang_vel", ("gaussian", 0.0, 0.2), (-10.0, 10.0), (0.5, 1.0, -2.0)),
    ("last_action", ("gaussian", 0.05, 0.15), (-1.0, 1.0), None),
    ("world_height_map", ("gaussian", 0.02, 0.05), (-0.3, 0.9), 2.0),
]
CRITIC = [                                                     # the critic's own clips and scales, no noise
    ("goal_relative_xyz", None, (-5.0, 5.0), None),
    ("root_euler_xyz", None, None, 0.5),
    ("base_lin_vel", None, (-10.0, 10.0), None),
    ("base_ang_vel", None, (-10.0, 10.0), (1.0, 2.0, 0.5)),
    ("last_action", None, (-1.0, 1.0), None),
    ("world_height_map", None, (-0.5, 0.5), 2.0),              # a narrow clip: misses (+inf) and high ground both clip
]
EXTRA = ["wheel_friction", "base_mass", "motor_damping"]      # 9 floats: Dc = 698


def _bits(x):
    return x.contiguous().view(torch.int32)


def _spec(n, seed=11, corrupt=1):
    spec = wl.elevation_task(num_envs=n, seed=seed)
    spec.cfg.enable_corruption = corrupt
    return spec


def _sim(spec, row_terms=None, critic=None, extra=(), scan=None):
    sim = WheeledSim(spec, DEV)
    if scan is not None:
        sim.set_scan_tma(scan)
    if row_terms is not None:
        sim.set_row_terms(row_terms)
    if critic is not None:
        sim.set_row_critic(critic, extra)
    sim.startup()
    sim.reset(None, 0)
    return sim


EXTRA_ODD = ["wheel_friction", "motor_damping"]               # 8 floats: Dc = 697, so N * Dc is odd for odd N


def _state_views(sim):
    from wheeledlab_b200.sim import G_PKD, G_PMU_D
    g = sim.groups
    return torch.cat([g[G_PMU_D], g[G_PKD]], dim=1)


# ---- 1. the critic row --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [1, 33, 4096])
@pytest.mark.parametrize("scan", [0, 1])
def test_critic_row_equals_the_twin_the_noise_free_row_and_the_state_views(n, scan):
    spec = _spec(n)
    noisy = _sim(spec, POLICY_GAUSS, CRITIC, EXTRA_ODD, scan)
    plain = _sim(_spec(n), CRITIC, CRITIC, EXTRA_ODD, scan)      # policy row = the critic's terms, no noise
    twin = R.RowOracle(spec.cfg, heightfield=spec.heightfield)
    twin.startup()
    assert noisy.critic_obs_dim == 697 and noisy.row_terms == 6
    assert (n * 697) % 2 == (n % 2)
    resets = 0

    def check(t, obs_n, obs_p):
        c, cp = noisy.critic_observe(), plain.critic_observe()
        assert torch.equal(_bits(c), _bits(cp)), ("the policy row's noise reached the critic", t)
        assert torch.equal(_bits(c[:, :D]), _bits(obs_p)), ("critic row != noise-free policy row", t)
        assert torch.equal(_bits(c[:, D:]), _bits(_state_views(noisy))), ("extra columns", t)
        twin.import_state(noisy.groups.cpu().numpy())
        assert np.array_equal(_bits(c[:, :D]).cpu().numpy(), twin.row_observe(CRITIC, t, -1).view(np.int32)), ("twin", t)
        assert torch.isfinite(c).all()
        assert not torch.equal(obs_n, obs_p)

    steps = 6 if n > 1000 else 30
    for t in range(steps):                                            # host counters
        act = noisy.synth_actions(t)
        obs_n, _, term, trunc = noisy.step(act, t)
        obs_p = plain.step(act, t)[0]
        resets += int((term | trunc).sum())
        check(t, obs_n, obs_p)
    for s in (noisy, plain):
        s.set_step_counter(steps)
    for k in range(2):                                                # device counters
        act = noisy.synth_actions(steps + k)
        t = WheeledSim.device_counter_plus(k)
        check(steps + k, noisy.step(act, t)[0], plain.step(act, t)[0])
    if n == 4096:
        assert resets > 0, "the steps reset some envs"


def test_critic_map_miss_is_clipped_like_the_policy_row():
    # an env whose scan window leaves the height-field: every miss is +inf before the clip, so the critic's map columns read
    # the clip bound times the scale, as the policy row does under the same term
    n = 8
    spec = _spec(n)
    sim = _sim(spec, CRITIC, CRITIC)
    from wheeledlab_b200.sim import G_POS
    g = sim.groups
    g[G_POS, 0, 0] = spec.cfg.hf_x0 - 5.0                            # env 0 far outside the raster
    g[G_POS, 0, 1] = spec.cfg.hf_y0 - 5.0
    obs = sim.observe(0, 0)
    c = sim.critic_observe()
    assert torch.equal(_bits(c[0, 13:D]), _bits(obs[0, 13:D]))
    assert torch.all(c[0, 13:D] == 0.5 * 2.0), "a miss is +inf, clipped to 0.5, scaled by 2"


def test_row_critic_refusals_leave_the_handle_as_it_was():
    spec = _spec(16)
    sim = _sim(spec, None, CRITIC, EXTRA)
    assert sim.critic_obs_dim == 698
    noisy = [CRITIC[0]] + [("root_euler_xyz", ("gaussian", 0.0, 0.1), None, None)] + CRITIC[2:]
    with pytest.raises(WlError, match="root_euler_xyz.*noise-free"):
        sim.set_row_critic(noisy)
    with pytest.raises(WlError, match="world_height_map.*clip"):
        sim.set_row_critic(CRITIC[:5] + [("world_height_map", None, None, 2.0)])
    with pytest.raises(WlError, match="kind"):
        sim.set_row_critic(CRITIC[1:] + CRITIC[:1])
    with pytest.raises(WlError, match="32 floats"):
        sim.set_row_critic(CRITIC, EXTRA * 4)
    assert sim.critic_obs_dim == 698
    with pytest.raises(WlError, match="Drift family"):
        sim.set_critic_terms(["root_pos_w"])
    for other in (wl.drift_task(num_envs=16, seed=1), wl.visual_task(num_envs=16, seed=1)):
        s = WheeledSim(other, DEV)
        with pytest.raises(WlError, match="Elevation"):
            s.set_row_critic(CRITIC)
        assert s.critic_obs_dim == 0
    assert sim.set_row_critic([]) == 0 and sim.critic_obs_dim == 0


# ---- 2. the wide asymmetric policy ---------------------------------------------------------------------------------------------
def _nets(seed, d, dc):
    torch.manual_seed(seed)
    mk = lambda nin, out: torch.nn.Sequential(torch.nn.Linear(nin, 64), torch.nn.ReLU(), torch.nn.Linear(64, 64), torch.nn.ReLU(),
                                              torch.nn.Linear(64, out)).to(DEV)
    return mk(d, 2), mk(dc, 1), torch.tensor((0.8, 1.2), device=DEV)


def _outs(n):
    return (torch.zeros(n, 2, device=DEV), torch.zeros(n, 2, device=DEV), torch.zeros(n, device=DEV), torch.zeros(n, device=DEV))


@pytest.mark.parametrize("n", [33, 4096])
@pytest.mark.parametrize("dc", [40, 698, 721])
def test_policy_act_wide_asym_equals_policy_act(n, dc):
    from wheeledlab_b200.policy import pack_actor_critic, policy_act, policy_act_wide_asym
    sim = _sim(_spec(n), POLICY_GAUSS)
    obs = sim.step(sim.synth_actions(0), 0)[0].clone()
    actor, critic, std = _nets(1, D, D)
    blob = pack_actor_critic(actor, critic, std, D, DEV)
    sim.set_step_counter(40)
    t = sim.device_counter_plus(2)
    ref, same = _outs(n), _outs(n)
    policy_act(sim, obs, blob, *ref, t, "relu")
    policy_act_wide_asym(sim, obs, obs, blob, *same, t)
    for a, b, name in zip(same, ref, ("actions", "mean", "log_prob", "value")):
        assert torch.equal(_bits(a), _bits(b)), f"critic row = policy row: {name}"
    _, cdc, _ = _nets(2, D, dc)
    blob_dc = pack_actor_critic(actor, cdc, std, D, DEV, critic_obs_dim=dc)
    cobs = 0.5 * torch.randn(n, dc, device=DEV)
    asym = _outs(n)
    policy_act_wide_asym(sim, obs, cobs, blob_dc, *asym, t)
    for a, b, name in zip(asym[:3], ref[:3], ("actions", "mean", "log_prob")):
        assert torch.equal(_bits(a), _bits(b)), f"Dc = {dc}: {name}"
    want = copy.deepcopy(cdc).double()(cobs.double()).squeeze(-1)
    got32 = copy.deepcopy(cdc)(cobs).squeeze(-1).double()
    e_kernel, e_torch = (asym[3].double() - want).abs().max().item(), (got32 - want).abs().max().item()
    assert e_kernel <= max(4 * e_torch, 1e-6 * max(1.0, want.abs().max().item())), (e_kernel, e_torch)


# ---- 3. the wide asymmetric update ---------------------------------------------------------------------------------------------
def _synthetic(n, dc, seed=0):
    from wheeledlab_b200.policy import pack_actor_critic
    actor, critic, std = _nets(seed, D, dc)
    blob = pack_actor_critic(actor, critic, std, D, DEV, critic_obs_dim=dc)
    g = torch.Generator(device=DEV).manual_seed(seed + 1)
    ap, cp = copy.deepcopy(actor), copy.deepcopy(critic)
    with torch.no_grad():
        for net in (ap, cp):
            for p in net.parameters():
                p.add_(0.15 * p.abs().mean() * torch.randn(p.shape, device=DEV, generator=g))
        sp = std * torch.tensor([1.15, 0.9], device=DEV)
        obs = torch.randn(n, D, device=DEV, generator=g)
        cobs = torch.randn(n, dc, device=DEV, generator=g)
        mu = ap(obs)
        val = cp(cobs).squeeze(-1) + 0.25 * torch.randn(n, device=DEV, generator=g)
        act = mu + sp * torch.randn(n, 2, device=DEV, generator=g)
        lp = torch.distributions.Normal(mu, sp).log_prob(act).sum(-1)
        ret = val + 0.5 * torch.randn(n, device=DEV, generator=g)
        adv = 0.3 + torch.randn(n, device=DEV, generator=g)
    slab = SimpleNamespace(obs_in=obs.contiguous(), critic_obs_in=cobs.contiguous().view(1, n, dc), actions=act.contiguous(),
                           values=val.contiguous(), log_prob=lp.contiguous(), mean=mu.contiguous())
    perm = torch.randperm(n, device=DEV, generator=g)
    return (actor, critic, std), blob, slab, ret.contiguous(), adv.contiguous(), perm


def test_update_wide_asym_on_the_policy_row_is_update_wide_bit_for_bit():
    from wheeledlab_b200.learner import FusedPPO, PPOConfig
    cfg = PPOConfig()
    n = 4096 * 4
    _, blob, slab, ret, adv, perm = _synthetic(n, D, seed=4)
    slab.critic_obs_in = slab.obs_in.view(1, n, D)
    b_sym, b_asym = blob.clone(), blob.clone()
    sym, asym = FusedPPO(b_sym, D, cfg, "relu"), FusedPPO(b_asym, D, cfg, "relu", critic_obs_dim=D)
    for _ in range(2):
        sym.update(slab, ret, adv, perm)
        asym.update(slab, ret, adv, perm)
    assert not torch.equal(b_sym, blob)
    for a, b, name in ((b_asym, b_sym, "blob"), (asym.m, sym.m, "m"), (asym.v, sym.v, "v"), (asym.state, sym.state, "state"),
                       (asym.last_gradient(), sym.last_gradient(), "gradient")):
        assert torch.equal(_bits(a), _bits(b)), name


def _loss(actor, critic, std, slab, ret, adv, cfg, dt):
    obs, cobs = slab.obs_in.to(dt), slab.critic_obs_in[0].to(dt)
    A = adv.to(dt)
    A = (A - A.mean()) / (A.std() + 1e-8)
    mu, V = actor(obs), critic(cobs).squeeze(-1)
    dist = torch.distributions.Normal(mu, std.expand_as(mu))
    ratio = torch.exp(dist.log_prob(slab.actions.to(dt)).sum(-1) - slab.log_prob.to(dt))
    surr = torch.max(-A * ratio, -A * ratio.clamp(1 - cfg.clip_param, 1 + cfg.clip_param)).mean()
    vo, R_ = slab.values.to(dt), ret.to(dt)
    vc = vo + (V - vo).clamp(-cfg.clip_param, cfg.clip_param)
    vl = torch.max((V - R_) ** 2, (vc - R_) ** 2).mean()
    return surr + cfg.value_loss_coef * vl - cfg.entropy_coef * dist.entropy().sum(-1).mean()


@pytest.mark.parametrize("dc", [40, 689, 698, 721])
def test_update_wide_asym_gradient_against_fp64(dc):
    from wheeledlab_b200.learner import FusedPPO, PPOConfig
    from wheeledlab_b200.policy import actor_critic_state_dict
    n = 8192
    nets, blob, slab, ret, adv, _ = _synthetic(n, dc, seed=dc)
    perm = torch.arange(n, device=DEV).flip(0).contiguous()     # rows are gathered through a permutation
    cfg = PPOConfig(num_learning_epochs=1, num_mini_batches=1)
    grads = {}
    for dt in (torch.float32, torch.float64):
        actor, critic = copy.deepcopy(nets[0]).to(dt), copy.deepcopy(nets[1]).to(dt)
        std = nets[2].to(dt).clone().requires_grad_(True)
        _loss(actor, critic, std, slab, ret, adv, cfg, dt).backward()
        sd = {f"actor.{k}": v.grad for k, v in actor.named_parameters()}
        sd.update({f"critic.{k}": v.grad for k, v in critic.named_parameters()})
        sd["std"] = std.grad
        grads[dt] = sd
    ppo = FusedPPO(blob, D, cfg, "relu", critic_obs_dim=dc)
    ppo.update(slab, ret, adv, perm)
    got = actor_critic_state_dict(ppo.last_gradient()[:blob.numel()], D, dc)
    assert got["critic.0.weight"].shape == (64, dc)
    for k, g64 in grads[torch.float64].items():
        scale = g64.abs().max().item()
        e_fused = (got[k].double() - g64).abs().max().item() / scale
        e_torch = (grads[torch.float32][k].double() - g64).abs().max().item() / scale
        assert e_fused <= max(4 * e_torch, 1e-6), f"d{k}: {e_fused:.3g} vs torch fp32 {e_torch:.3g}"


def test_update_wide_asym_never_steps_the_padding_and_replays_reproducibly():
    from wheeledlab_b200.learner import FusedPPO, PPOConfig
    from wheeledlab_b200.policy import blob_layout
    dc = 698                                                   # two padding rows in the critic's W1t, three in the actor's
    cfg = PPOConfig(num_learning_epochs=2, num_mini_batches=4)
    _, blob, slab, ret, adv, perm = _synthetic(4096 * 4, dc, seed=9)
    off, total = blob_layout(D, dc)
    lens = [D * 64, 64, 4096, 64, 128, 2, dc * 64, 64, 4096, 64, 64, 1, 2]
    pad = torch.ones(total, dtype=torch.bool)
    for o, k in zip(off, lens):
        pad[o:o + k] = False
    pad = pad.to(DEV)
    runs = []
    for capture in (False, True):
        b = blob.clone()
        ppo = FusedPPO(b, D, cfg, "relu", critic_obs_dim=dc)
        if capture:
            ppo._workspace(perm.numel())
            s = torch.cuda.Stream()
            s.wait_stream(torch.cuda.current_stream())
            g = torch.cuda.CUDAGraph()
            with torch.cuda.stream(s), torch.cuda.graph(g, stream=s):
                ppo.update(slab, ret, adv, perm)
            g.replay()
        else:
            ppo.update(slab, ret, adv, perm)
        torch.cuda.synchronize()
        runs.append((b, ppo.m.clone(), ppo.v.clone(), ppo.state.clone()))
    for x in runs[0][:3]:
        assert not torch.any(x[pad] != 0)
    assert not torch.equal(runs[0][0], blob)
    for a, b in zip(*runs):
        assert torch.equal(_bits(a), _bits(b))


def test_update_wide_asym_refusals():
    from wheeledlab_b200._lib import lib
    from wheeledlab_b200.learner import FusedPPO, PPOConfig
    assert lib.wl_ppo_wide_asym_workspace_bytes(D, 0, 4096, 4) == 0 and b"critic_obs_dim" in lib.wl_last_error()
    assert lib.wl_ppo_wide_asym_workspace_bytes(D, 4097, 4096, 4) == 0
    assert lib.wl_ppo_wide_asym_workspace_bytes(D, 698, 4096, 4) > lib.wl_ppo_wide_workspace_bytes(D, 4096, 4) - 4096 * 4
    with pytest.raises(NotImplementedError, match="relu"):
        FusedPPO(torch.zeros(12000, device=DEV), 14, PPOConfig(), activation="relu", critic_obs_dim=20)


# ---- 4. the iteration and the runner --------------------------------------------------------------------------------------------
def _iteration(n, T, policy_terms, critic_terms, extra, capture, critic=True, seed=2):
    from wheeledlab_b200.learner import PPOConfig, PPOIteration
    from wheeledlab_b200.policy import pack_actor_critic
    sim = _sim(_spec(n, seed=seed), policy_terms, critic_terms if critic else None, extra)
    dc = sim.critic_obs_dim if critic else None
    actor, crit, _ = _nets(seed, D, dc or D)
    blob = pack_actor_critic(actor, crit, torch.ones(2, device=DEV), D, DEV, critic_obs_dim=dc)
    it = PPOIteration(sim, blob, PPOConfig(), T, "relu", episode_stats=True, critic=critic).start(0, capture=capture)
    return it, blob


def _perms(n, k):
    g = torch.Generator(device=DEV).manual_seed(123)
    return [torch.randperm(n, device=DEV, generator=g) for _ in range(k)]


def test_iteration_is_one_graph_and_equals_eager():
    n, T = 256, 16
    cap, blob_c = _iteration(n, T, POLICY_GAUSS, CRITIC, EXTRA, capture=True)
    eag, blob_e = _iteration(n, T, POLICY_GAUSS, CRITIC, EXTRA, capture=False)
    assert cap.graph is not None and cap.roll.graph is None
    launches = cap.sim.launch_count
    for p in _perms(n * T, 2):
        cap.run(p)
        eag.run(p)
    assert cap.sim.launch_count == launches
    torch.cuda.synchronize()
    slab = cap.roll.slab
    assert slab.critic_obs_in.shape == (T + 1, n, 698)
    for a, b, name in ((blob_c, blob_e, "blob"), (cap.ppo.m, eag.ppo.m, "m"), (cap.ppo.state, eag.ppo.state, "state"),
                       (slab.flat, eag.roll.slab.flat, "slab"), (slab.critic_obs_in, eag.roll.slab.critic_obs_in, "critic_obs_in"),
                       (cap.sim.groups, eag.sim.groups, "env state")):
        assert torch.equal(a.view(torch.uint8), b.view(torch.uint8)), name
    from wheeledlab_b200.policy import critic_value
    want = critic_value(blob_c, D, slab.critic_obs_in[T], "relu", 698)
    assert torch.equal(_bits(cap._bootstrap()), _bits(want)), "the bootstrap reads the critic row"
    assert not torch.equal(slab.critic_obs_in[T][:, :D], slab.obs[T - 1]), "the policy row is noisy, the critic row is not"


def test_iteration_on_the_policy_row_equals_the_symmetric_one():
    n, T = 256, 16
    asym, blob_a = _iteration(n, T, CRITIC, CRITIC, (), capture=True)
    sym, blob_s = _iteration(n, T, CRITIC, None, (), capture=True, critic=False)
    assert torch.equal(blob_a, blob_s)
    for p in _perms(n * T, 2):
        asym.run(p)
        sym.run(p)
    torch.cuda.synchronize()
    assert torch.equal(asym.roll.slab.critic_obs_in[:T], asym.roll.slab.obs_in)
    for a, b, name in ((blob_a, blob_s, "blob"), (asym.ppo.m, sym.ppo.m, "m"), (asym.ppo.state, sym.ppo.state, "state"),
                       (asym.roll.slab.flat, sym.roll.slab.flat, "slab"), (asym.sim.groups, sym.sim.groups, "env state")):
        assert torch.equal(a.view(torch.uint8), b.view(torch.uint8)), name


def _agent_cfg(save_interval=1, T=16):
    from dataclasses import asdict
    from wheeledlab_b200.learner import PPOConfig
    return {"num_steps_per_env": T, "save_interval": save_interval, "empirical_normalization": False,
            "policy": {"class_name": "ActorCritic", "init_noise_std": 1.0, "actor_hidden_dims": [64, 64], "critic_hidden_dims": [64, 64],
                       "activation": "relu"},
            "algorithm": {"class_name": "PPO", **asdict(PPOConfig())}}


def _env(n, critic=True):
    spec = wl.make_task("Isaac-MushrElevationRL-v0", num_envs=n, seed=4)
    spec.cfg.enable_corruption = 1
    env = wl.ManagerBasedRLEnv(spec, device=DEV)
    env.set_row_terms([(name, name, {"noise": nz, "clip": cl, "scale": sc}) for name, nz, cl, sc in POLICY_GAUSS])
    if critic:
        env.set_critic_observation([(name, name, {"clip": cl, "scale": sc}) for name, _, cl, sc in CRITIC] + EXTRA)
    return env


def test_env_routes_a_row_critic_group():
    env = _env(32)
    assert env.observation_manager.group_obs_dim["critic"] == (698,)
    obs, rew, term, trunc, extras = env.step(env.sim.synth_actions(0))
    c = extras["observations"]["critic"]
    assert c.shape == (32, 698) and torch.equal(_bits(c), _bits(env.sim.critic_observe()))
    with pytest.raises(WlError, match="Drift family"):
        env.set_critic_observation(["root_pos_w"])                # a library-only group keeps today's refusal
    with pytest.raises(NotImplementedError, match="noise"):
        env.set_critic_observation([(name, name, {"noise": ("gaussian", 0.0, 0.1)}) for name, _, _, _ in CRITIC])
    assert env.observation_manager.group_obs_dim["critic"] == (698,)


def test_runner_trains_saves_loads_resumes_and_plays(tmp_path):
    from wheeledlab_b200.learner import FusedOnPolicyRunner, PPOIteration
    torch.manual_seed(1)
    env = _env(256)
    cfg = _agent_cfg()
    a = FusedOnPolicyRunner(env, cfg, log_dir=str(tmp_path), device=DEV)
    assert type(a.it) is PPOIteration and a.it.graph is None and a.critic_obs_dim == 698
    a.learn(3)
    assert a.it.graph is not None and a.it.roll.graph is None
    ck = torch.load(tmp_path / "models" / "model_2.pt")
    assert ck["model_state_dict"]["critic.0.weight"].shape == (64, 698)
    assert ck["model_state_dict"]["actor.0.weight"].shape == (64, D)
    kept = str(tmp_path / "kept.pt")
    torch.save(ck, kept)
    b = FusedOnPolicyRunner(env, cfg, device=DEV)
    b.load(kept)
    for x, y in ((a.blob, b.blob), (a.alg.m, b.alg.m), (a.alg.v, b.alg.v)):
        assert torch.equal(_bits(x), _bits(y))
    a.alg.state[0] = cfg["algorithm"]["learning_rate"]
    a.learn(1)
    b.it.roll.slab, b.it.roll.obs0, b.it.roll.cobs0 = a.it.roll.slab, a.it.roll.obs0, a.it.roll.cobs0
    b.it.perm.copy_(a.it.perm)
    b.it._learn()
    torch.cuda.synchronize()
    for name, x, y in (("blob", a.blob, b.blob), ("m", a.alg.m, b.alg.m), ("v", a.alg.v, b.alg.v)):
        assert torch.equal(_bits(x), _bits(y)), name
    # another critic width is refused before anything is written; an env without the group plays the actor alone
    plain = FusedOnPolicyRunner(_env(256, critic=False), cfg, device=DEV)
    before = plain.blob.clone()
    with pytest.raises(ValueError, match="critic.0"):
        plain.load(kept)
    assert torch.equal(before, plain.blob)
    plain.load(kept, load_optimizer=False)
    c = FusedOnPolicyRunner(env, cfg, device=DEV)
    c.load(kept)
    obs = a.it.roll.slab.obs_in[2]
    assert torch.equal(_bits(plain.get_inference_policy()(obs)), _bits(c.get_inference_policy()(obs)))
