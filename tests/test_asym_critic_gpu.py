"""The asymmetric actor-critic on the device (DESIGN 6m): wl_critic_observe against the policy row and the state views,
wl_policy_act_asym against wl_policy_act_elu and fp64, wl_ppo_update_asym against wl_ppo_update (bit for bit when the critic
reads the policy row) and against fp64 autograd, and the one-graph iteration built on them."""
import copy
import ctypes as C
import itertools
from types import SimpleNamespace

import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
D = 14
LIBRARY = ["root_pos_w", "root_euler_xyz", "base_lin_vel", "base_ang_vel", "last_action", "joint_vel", "joint_pos", "wheel_friction",
           "base_mass", "motor_damping"]
POLICY_TERMS = ["root_pos_w", "root_euler_xyz", "base_lin_vel", "base_ang_vel", ("last_action", 1.0)]
SIZES = [1, 31, 33, 4096, 33793]


def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")


def _bits(x):
    return x.contiguous().view(torch.int32)


def _same_values_and_bits(a, b, what):
    """Equal as fp32 values everywhere, and bit for bit wherever the value is not a zero (the policy row's "+ 0 * z" may turn
    a -0 into +0)."""
    assert torch.equal(a, b), what
    nz = a != 0
    assert torch.equal(_bits(a)[nz], _bits(b)[nz]), what


def _sim(task, n, seed=5, noise=False, offset=0):
    import wheeledlab_b200 as wl
    spec = wl.make_task(task, num_envs=n, seed=seed, env_id_offset=offset)
    if not noise:
        for k in range(4):
            spec.cfg.noise_std[k] = 0.0
    sim = wl.WheeledSim(spec, DEV)
    sim.startup()
    sim.reset(None, 0)
    return sim


def _expected_columns(sim):
    from wheeledlab_b200.sim import G_PKD, G_PMASS, G_PMU_D
    g = sim.groups
    return {"joint_vel": sim.wheel_vel, "joint_pos": sim.steer_pos, "wheel_friction": g[G_PMU_D], "base_mass": g[G_PMASS, :, 0:1],
            "motor_damping": g[G_PKD]}


@pytest.mark.parametrize("task", ["drift", "f1tenth_drift", "hound_4wd"])
@pytest.mark.parametrize("n", SIZES)
def test_critic_observe_equals_the_noise_free_policy_row_and_the_state_views(task, n):
    _need_gpu()
    sim = _sim(task, n)
    assert sim.set_critic_terms(POLICY_TERMS + LIBRARY[5:]) == 29
    steps = 40 if n > 4096 else 230                        # 230 steps cross time-outs, off-track resets and pushes
    resets = 0
    for t in range(steps):
        obs, _, term, trunc = sim.step(sim.synth_actions(t), t)
        resets += int((term | trunc).sum())
        if t % 7 == 0 or t == steps - 1:
            c = sim.critic_observe()
            _same_values_and_bits(c[:, :14], obs, f"{task} n={n} step {t}: shared columns")
            col = 14
            for name, want in _expected_columns(sim).items():
                w = want.shape[1]
                assert torch.equal(_bits(c[:, col:col + w]), _bits(want)), f"{task} n={n} step {t}: {name}"
                col += w
    if n >= 31 and steps == 230:
        assert resets > 0, "the trajectory crossed no reset"


def test_critic_observe_leaves_the_noise_out():
    """With the reference's noise on, the critic row is the row a noise-0 handle with the same state forms."""
    _need_gpu()
    noisy, clean = _sim("drift", 4096, noise=True), _sim("drift", 4096)
    for s in (noisy, clean):
        s.set_critic_terms(POLICY_TERMS)
    for t in range(12):
        act = noisy.synth_actions(t)
        obs_noisy, *_ = noisy.step(act, t)
        obs_clean, *_ = clean.step(act, t)
    assert torch.equal(noisy.groups, clean.groups), "noise is observation-only"
    assert not torch.equal(obs_noisy, obs_clean)
    assert torch.equal(_bits(noisy.critic_observe()), _bits(clean.critic_observe()))
    _same_values_and_bits(noisy.critic_observe(), obs_clean, "critic row vs the noise-free policy row")


def test_critic_observe_every_subset_and_order_offset_and_replacement():
    _need_gpu()
    n = 33
    sim = _sim("drift", n, offset=1000)
    for t in range(9):
        sim.step(sim.synth_actions(t), t)
    from wheeledlab_b200._lib import WL_CRITIC_TERMS
    assert sim.set_critic_terms(LIBRARY) == 29
    full = sim.critic_observe()
    first, col = {}, 0
    for name in LIBRARY:
        first[name] = col
        col += WL_CRITIC_TERMS[name][1]
    torch.manual_seed(0)
    tables = [list(c) for r in range(1, 4) for c in itertools.combinations(LIBRARY, r)]
    tables += [[LIBRARY[i] for i in torch.randperm(10).tolist()[:k]] for k in range(4, 11) for _ in range(6)]
    for names in tables:                                    # a table replaced between calls
        dc = sim.set_critic_terms(names)
        want = torch.cat([full[:, first[x]:first[x] + WL_CRITIC_TERMS[x][1]] for x in names], dim=1)
        assert dc == want.shape[1]
        assert torch.equal(_bits(sim.critic_observe()), _bits(want)), names
    # an unaligned output (a slab row of an odd N * Dc) and the clip
    sim.set_critic_terms(["base_mass", ("joint_vel", 0.5)])
    buf = torch.zeros(n * 5 + 1, device=DEV)
    out = buf[1:].view(n, 5)
    sim.critic_observe(out=out)
    assert torch.equal(out[:, 0:1], full[:, first["base_mass"]:first["base_mass"] + 1])
    assert torch.equal(out[:, 1:], full[:, first["joint_vel"]:first["joint_vel"] + 4].clamp(-0.5, 0.5)) and buf[0] == 0


def test_critic_table_refusals_leave_the_handle_as_it_was():
    _need_gpu()
    import wheeledlab_b200 as wl
    from wheeledlab_b200._lib import WlCriticTerm, lib
    sim = _sim("drift", 8)
    assert sim.critic_obs_dim == 0
    out = torch.full((8, 3), 7.0, device=DEV)
    with pytest.raises(wl.WlError, match="no critic table"):
        sim.critic_observe(out=out)
    sim.set_critic_terms(["root_pos_w"])
    bad = [([(99, 0.0)], b"unknown term kind"), ([(1, -1.0)], b"clip"), ([(1, float("nan"))], b"clip"),
           ([(6, 0.0)] * 9, b"wider than 32")]
    for terms, msg in bad:
        arr = (WlCriticTerm * len(terms))(*[WlCriticTerm(k, c) for k, c in terms])
        assert lib.wl_set_critic_terms(sim._h, arr, len(terms)) == -1 and msg in lib.wl_last_error()
        assert sim.critic_obs_dim == 3
    assert lib.wl_set_critic_terms(sim._h, None, 2) == -1 and lib.wl_set_critic_terms(sim._h, None, 17) == -1
    assert lib.wl_critic_observe(sim._h, None, None) == -1
    assert torch.all(out == 7.0)
    elev = wl.WheeledSim(wl.elevation_task(num_envs=8, seed=1), DEV)
    arr = (WlCriticTerm * 1)(WlCriticTerm(1, 0.0))
    assert lib.wl_set_critic_terms(elev._h, arr, 1) == -3 and b"Drift family" in lib.wl_last_error()
    assert sim.set_critic_terms([]) == 0


# ---- wl_policy_act_asym ---------------------------------------------------------------------------------------------------

def _nets(seed, dc, std=(0.8, 1.2)):
    torch.manual_seed(seed)
    mk = lambda nin, out: torch.nn.Sequential(torch.nn.Linear(nin, 64), torch.nn.ELU(), torch.nn.Linear(64, 64), torch.nn.ELU(),
                                              torch.nn.Linear(64, out)).to(DEV)
    return mk(D, 2), mk(dc, 1), torch.tensor(std, device=DEV)


def _outs(n):
    return (torch.zeros(n, 2, device=DEV), torch.zeros(n, 2, device=DEV), torch.zeros(n, device=DEV), torch.zeros(n, device=DEV))


@pytest.mark.parametrize("n", SIZES)
@pytest.mark.parametrize("device_counter", [False, True])
def test_policy_act_asym_equals_policy_act_elu(n, device_counter):
    _need_gpu()
    from wheeledlab_b200.policy import pack_actor_critic, policy_act, policy_act_asym
    sim = _sim("drift", n, noise=True, offset=77)
    actor, critic, std = _nets(1, D)
    blob = pack_actor_critic(actor, critic, std, D, DEV)
    assert torch.equal(blob, pack_actor_critic(actor, critic, std, D, DEV, critic_obs_dim=D))
    obs = sim.observe(0)
    if device_counter:
        sim.set_step_counter(40)
        t = sim.device_counter_plus(2)
    else:
        t = 42
    ref, sym = _outs(n), _outs(n)
    policy_act(sim, obs, blob, *ref, t, "elu")
    policy_act_asym(sim, obs, obs, blob, *sym, t)
    for a, b, name in zip(sym, ref, ("actions", "mean", "log_prob", "value")):
        assert torch.equal(_bits(a), _bits(b)), f"critic row = policy row: {name}"
    # another critic input and width: the actor's three outputs do not move
    _, critic29, _ = _nets(2, 29)
    blob29 = pack_actor_critic(actor, critic29, std, D, DEV, critic_obs_dim=29)
    asym = _outs(n)
    policy_act_asym(sim, obs, torch.randn(n, 29, device=DEV), blob29, *asym, t)
    for a, b, name in zip(asym[:3], ref[:3], ("actions", "mean", "log_prob")):
        assert torch.equal(_bits(a), _bits(b)), f"Dc = 29: {name}"
    assert not torch.equal(asym[3], ref[3])


@pytest.mark.parametrize("dc", [1, 17, 29, 32])
def test_policy_act_asym_value_against_fp64(dc):
    _need_gpu()
    from wheeledlab_b200.policy import critic_value, pack_actor_critic, policy_act_asym
    n = 4096
    sim = _sim("drift", n)
    actor, critic, std = _nets(3, dc)
    blob = pack_actor_critic(actor, critic, std, D, DEV, critic_obs_dim=dc)
    cobs = 2.0 * torch.randn(n, dc, device=DEV)
    out = _outs(n)
    policy_act_asym(sim, sim.observe(0), cobs, blob, *out, 3)
    want = copy.deepcopy(critic).double()(cobs.double()).squeeze(-1)
    # the act step's ELU criterion: __expf in the kernel, 1e-5 of the value scale
    assert (out[3].double() - want).abs().max().item() <= 1e-5 * max(1.0, want.abs().max().item())
    assert torch.allclose(critic_value(blob, D, cobs, critic_obs_dim=dc).double(), want, rtol=1e-4, atol=1e-5)


def test_policy_act_asym_refusals_leave_outputs_untouched():
    _need_gpu()
    from wheeledlab_b200._lib import WlPolicyOut, lib
    from wheeledlab_b200.policy import blob_layout
    n = 33
    sim = _sim("drift", n)
    obs, cobs = sim.observe(0), torch.zeros(n, 17, device=DEV)
    blob = torch.zeros(blob_layout(D, 17)[1], device=DEV)
    outs = [torch.full_like(x, 7.0) for x in _outs(n)]
    po = WlPolicyOut(*[x.data_ptr() for x in outs])
    p = lambda x: C.c_void_p(x.data_ptr())
    call = lambda o, c, dc, b, po_, t: lib.wl_policy_act_asym(sim._h, o, c, dc, b, po_, t, None)
    assert call(p(obs), p(cobs), 0, p(blob), po, 0) == -1 and b"critic_obs_dim" in lib.wl_last_error()
    assert call(p(obs), p(cobs), 33, p(blob), po, 0) == -1
    assert call(p(obs), None, 17, p(blob), po, 0) == -1
    assert call(None, p(cobs), 17, p(blob), po, 0) == -1
    assert call(p(obs), p(cobs), 17, C.c_void_p(blob.data_ptr() + 4), po, 0) == -1
    assert call(p(obs), C.c_void_p(cobs.data_ptr() + 2), 17, p(blob), po, 0) == -1
    assert call(p(obs), p(cobs), 17, p(blob), po, 1 << 31) == -1
    assert call(p(obs), p(cobs), 17, p(blob), WlPolicyOut(outs[0].data_ptr(), outs[1].data_ptr(), outs[2].data_ptr(), None), 0) == -1
    torch.cuda.synchronize()
    assert all(torch.all(x == 7.0) for x in outs)


# ---- wl_ppo_update_asym -----------------------------------------------------------------------------------------------------

def _synthetic(n, dc, seed=0):
    """tests/test_ppo_update_gpu.py's synthetic batch with a critic row of its own: ratios on both sides of the clip range,
    value changes on both sides of the value clip."""
    from wheeledlab_b200.policy import pack_actor_critic
    actor, critic, std = _nets(seed, dc)
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


@pytest.mark.parametrize("schedule", ["adaptive", "fixed"])
def test_update_asym_with_the_policy_row_is_update_bit_for_bit(schedule):
    _need_gpu()
    from wheeledlab_b200.learner import FusedPPO, PPOConfig
    cfg = PPOConfig(schedule=schedule)
    n = 4096 * 16
    _, blob, slab, ret, adv, perm = _synthetic(n, D, seed=4)
    slab.critic_obs_in = slab.obs_in.view(1, n, D)
    b_sym, b_asym = blob.clone(), blob.clone()
    sym, asym = FusedPPO(b_sym, D, cfg), FusedPPO(b_asym, D, cfg, critic_obs_dim=D)
    for _ in range(2):
        sym.update(slab, ret, adv, perm)
        asym.update(slab, ret, adv, perm)
    assert not torch.equal(b_sym, blob)
    for a, b, name in ((b_asym, b_sym, "blob"), (asym.m, sym.m, "m"), (asym.v, sym.v, "v"), (asym.state, sym.state, "state"),
                       (asym.history, sym.history, "history"), (asym.last_gradient(), sym.last_gradient(), "gradient")):
        assert torch.equal(_bits(a), _bits(b)), name


def _loss(actor, critic, std, slab, ret, adv, cfg, dt):
    """rsl_rl PPO.update()'s loss on one mini-batch = the whole batch, with privileged critic observations."""
    obs, cobs = slab.obs_in.to(dt), slab.critic_obs_in[0].to(dt)
    A = adv.to(dt)
    A = (A - A.mean()) / (A.std() + 1e-8)
    mu, V = actor(obs), critic(cobs).squeeze(-1)
    dist = torch.distributions.Normal(mu, std.expand_as(mu))
    ratio = torch.exp(dist.log_prob(slab.actions.to(dt)).sum(-1) - slab.log_prob.to(dt))
    surr = torch.max(-A * ratio, -A * ratio.clamp(1 - cfg.clip_param, 1 + cfg.clip_param)).mean()
    vo, R = slab.values.to(dt), ret.to(dt)
    vc = vo + (V - vo).clamp(-cfg.clip_param, cfg.clip_param)
    vl = torch.max((V - R) ** 2, (vc - R) ** 2).mean()
    return surr + cfg.value_loss_coef * vl - cfg.entropy_coef * dist.entropy().sum(-1).mean()


@pytest.mark.parametrize("dc", [17, 29])
def test_update_asym_gradient_against_fp64_per_element(dc):
    _need_gpu()
    from wheeledlab_b200.learner import FusedPPO, PPOConfig
    from wheeledlab_b200.policy import actor_critic_state_dict
    n = 16384
    nets, blob, slab, ret, adv, _ = _synthetic(n, dc, seed=dc)
    perm = torch.arange(n, device=DEV).flip(0).contiguous()     # a permutation that is not the identity: rows are gathered
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
    ppo = FusedPPO(blob, D, cfg, critic_obs_dim=dc)
    ppo.update(slab, ret, adv, perm)
    got = actor_critic_state_dict(ppo.last_gradient()[:blob.numel()], D, dc)
    assert got["critic.0.weight"].shape == (64, dc)
    for k, g64 in grads[torch.float64].items():
        scale = g64.abs().max().item()
        e_fused = (got[k].double() - g64).abs().max().item() / scale
        e_torch = (grads[torch.float32][k].double() - g64).abs().max().item() / scale
        assert e_fused <= max(4 * e_torch, 1e-6), f"d{k}: {e_fused:.3g} vs torch fp32 {e_torch:.3g}"


def _padding_mask(dc):
    from wheeledlab_b200.policy import blob_layout
    off, total = blob_layout(D, dc)
    lens = [D * 64, 64, 4096, 64, 128, 2, dc * 64, 64, 4096, 64, 64, 1, 2]
    m = torch.ones(total, dtype=torch.bool)
    for o, k in zip(off, lens):
        m[o:o + k] = False
    return m.to(DEV)


def test_update_asym_never_steps_the_padding_and_is_reproducible():
    _need_gpu()
    from wheeledlab_b200.learner import FusedPPO, PPOConfig
    dc = 29                                                    # three padding rows in the critic's W1t
    cfg = PPOConfig(num_learning_epochs=5, num_mini_batches=4)    # 20 mini-batches
    _, blob, slab, ret, adv, perm = _synthetic(4096 * 8, dc, seed=9)
    runs = []
    for _ in range(2):
        b = blob.clone()
        ppo = FusedPPO(b, D, cfg, critic_obs_dim=dc)
        ppo.update(slab, ret, adv, perm)
        runs.append((b, ppo.m.clone(), ppo.v.clone(), ppo.state.clone()))
    pad = _padding_mask(dc)
    assert int(pad.sum()) > 3 * 64
    for x in runs[0][:3]:
        assert not torch.any(x[pad] != 0)
    assert not torch.equal(runs[0][0], blob)
    for a, b in zip(*runs):
        assert torch.equal(_bits(a), _bits(b))


def test_update_asym_refusals():
    _need_gpu()
    from wheeledlab_b200._lib import lib
    from wheeledlab_b200.learner import FusedPPO, PPOConfig
    assert lib.wl_ppo_asym_workspace_bytes(14, 0, 4096, 4) == 0 and b"critic_obs_dim" in lib.wl_last_error()
    assert lib.wl_ppo_asym_workspace_bytes(14, 33, 4096, 4) == 0
    assert lib.wl_ppo_asym_workspace_bytes(17, 20, 4096, 4) == 0
    blob = torch.zeros(12000, device=DEV)
    with pytest.raises(NotImplementedError, match="relu"):
        FusedPPO(blob, D, PPOConfig(), activation="relu", critic_obs_dim=20)
    with pytest.raises(NotImplementedError, match="data-parallel"):
        FusedPPO(blob, D, PPOConfig(), exchange=object(), critic_obs_dim=20)
    _, b, slab, ret, adv, perm = _synthetic(4096, 20)
    before = b.clone()
    slab.critic_obs_in = None
    with pytest.raises(ValueError, match="critic_obs_in"):
        FusedPPO(b, D, PPOConfig(), critic_obs_dim=20).update(slab, ret, adv, perm)
    assert torch.equal(b, before)


# ---- the rollout and the iteration --------------------------------------------------------------------------------------------

def _iteration(n, T, terms, capture, seed=2, noise=True, critic=True):
    from wheeledlab_b200.learner import PPOConfig, PPOIteration
    from wheeledlab_b200.policy import pack_actor_critic
    sim = _sim("drift", n, seed=seed, noise=noise)
    dc = sim.set_critic_terms(terms) if critic else None
    actor, crit, _ = _nets(seed, dc if critic else D)
    blob = pack_actor_critic(actor, crit, torch.ones(2, device=DEV), D, DEV, critic_obs_dim=dc)
    it = PPOIteration(sim, blob, PPOConfig(), T, episode_stats=True, critic=critic).start(0, capture=capture)
    return it, blob, (actor, crit)


def _perms(n, k):
    g = torch.Generator(device=DEV).manual_seed(123)
    return [torch.randperm(n, device=DEV, generator=g) for _ in range(k)]


def test_asymmetric_iteration_is_one_graph_and_equals_eager():
    _need_gpu()
    n, T = 512, 24
    terms = POLICY_TERMS + ["wheel_friction", "base_mass", "motor_damping"]
    cap, blob_c, _ = _iteration(n, T, terms, capture=True)
    eag, blob_e, _ = _iteration(n, T, terms, capture=False)
    assert cap.graph is not None and cap.roll.graph is None and eag.graph is None
    launches = cap.sim.launch_count
    for p in _perms(n * T, 3):
        cap.run(p)
        eag.run(p)
    assert cap.sim.launch_count == launches, "the captured iteration launches nothing outside its graph"
    torch.cuda.synchronize()
    assert cap.roll.slab.critic_obs_in.shape == (T + 1, n, 23)
    pairs = [(blob_c, blob_e, "blob"), (cap.ppo.m, eag.ppo.m, "m"), (cap.ppo.v, eag.ppo.v, "v"), (cap.ppo.state, eag.ppo.state, "state"),
             (cap.roll.slab.flat, eag.roll.slab.flat, "slab"), (cap.roll.slab.critic_obs_in, eag.roll.slab.critic_obs_in, "critic_obs_in"),
             (cap.sim.groups, eag.sim.groups, "env state"), (cap.readback, eag.readback, "episode statistics")]
    for a, b, name in pairs:
        assert torch.equal(a.view(torch.uint8), b.view(torch.uint8)), name
    # the slab's critic rows are the rows the values were computed from, and row T is the bootstrap row
    slab = cap.roll.slab
    assert torch.equal(slab.critic_obs_in[T], cap.roll.cobs0) and torch.equal(cap.sim.critic_observe(), cap.roll.cobs0)
    assert torch.equal(slab.critic_obs_in[1:, :, 14:18], slab.critic_obs_in[:-1, :, 14:18]), "the DR columns are per env"


def test_bootstrap_value_is_taken_from_the_last_critic_row():
    _need_gpu()
    from wheeledlab_b200.policy import critic_value
    n, T = 256, 8
    it, blob, _ = _iteration(n, T, POLICY_TERMS, capture=False)            # noise on: the policy row differs from the critic row
    it.run(_perms(n * T, 1)[0])
    slab = it.roll.slab
    want = critic_value(blob, D, slab.critic_obs_in[T], critic_obs_dim=14)
    assert torch.equal(_bits(it._bootstrap()), _bits(want))
    assert not torch.equal(slab.critic_obs_in[T], slab.obs[T - 1]) and not torch.equal(want, critic_value(blob, D, slab.obs[T - 1]))


def test_asymmetric_iteration_on_the_policy_row_equals_the_symmetric_one():
    _need_gpu()
    n, T = 512, 24
    asym, blob_a, _ = _iteration(n, T, POLICY_TERMS, capture=True, noise=False)
    sym, blob_s, _ = _iteration(n, T, POLICY_TERMS, capture=True, noise=False, critic=False)
    assert torch.equal(blob_a, blob_s)
    for p in _perms(n * T, 3):
        asym.run(p)
        sym.run(p)
    torch.cuda.synchronize()
    assert torch.equal(asym.roll.slab.critic_obs_in[:T], asym.roll.slab.obs_in), "critic rows = policy rows on a noise-0 env"
    for a, b, name in ((blob_a, blob_s, "blob"), (asym.ppo.m, sym.ppo.m, "m"), (asym.ppo.state, sym.ppo.state, "state"),
                       (asym.roll.slab.flat, sym.roll.slab.flat, "slab"), (asym.readback, sym.readback, "episode statistics"),
                       (asym.sim.groups, sym.sim.groups, "env state")):
        assert torch.equal(a.view(torch.uint8), b.view(torch.uint8)), name


def test_asymmetric_checkpoint_round_trip_and_playback():
    """The blob as an rsl_rl state dict: critic.0.weight is [64, Dc]; a torch critic built from it reproduces slab.values;
    the actor plays through InferencePolicy and a deterministic rollout laid out for the symmetric network."""
    _need_gpu()
    from wheeledlab_b200.policy import (FusedPolicyRollout, InferencePolicy, actor_critic_state_dict, blob_layout,
                                        load_actor_critic_state_dict)
    n, T = 256, 16
    it, blob, _ = _iteration(n, T, LIBRARY, capture=True)
    it.run(_perms(n * T, 1)[0])
    sd = actor_critic_state_dict(blob, D, 29)
    assert sd["critic.0.weight"].shape == (64, 29) and sd["actor.0.weight"].shape == (64, D)
    actor, critic, _ = _nets(0, 29)
    torch.nn.ModuleDict({"actor": actor, "critic": critic}).load_state_dict({k: v for k, v in sd.items() if k != "std"})
    assert torch.equal(load_actor_critic_state_dict(sd, D, device=DEV, critic_obs_dim=29), blob)
    wrong = blob.clone()
    with pytest.raises(ValueError, match="critic.0"):
        load_actor_critic_state_dict(sd, D, out=wrong, critic_obs_dim=17)      # (a blob of the wrong layout, untouched)
    assert torch.equal(wrong, blob)
    # it.roll.slab.values were computed by the weights before the update: roll out again under the trained blob
    roll = FusedPolicyRollout(it.sim, blob, T, critic=True).capture(it.roll._base)
    slab = roll.run()
    want = critic.double()
    critic.load_state_dict({k[7:]: v.double() for k, v in actor_critic_state_dict(blob, D, 29).items() if k.startswith("critic.")})
    v64 = want(slab.critic_obs_in[:T].double()).squeeze(-1)
    assert (slab.values.double() - v64).abs().max().item() <= 1e-5 * max(1.0, v64.abs().max().item())
    # playback reads the actor only, and its blocks sit at the same offsets in both layouts: the asymmetric blob plays as it
    # is, and the unchanged checkpoint loads its actor into a blob of the symmetric layout
    off_a, _ = blob_layout(D, 29)
    off_s, total_s = blob_layout(D)
    assert off_a[:6] == off_s[:6]
    obs = slab.obs_in[3]
    assert torch.equal(_bits(InferencePolicy(blob, D, critic_obs_dim=29)(obs)), _bits(slab.mean[3]))
    with pytest.raises(ValueError, match="critic.0"):
        load_actor_critic_state_dict(sd, D, device=DEV)
    play = load_actor_critic_state_dict(sd, D, device=DEV, actor_only=True)
    assert play.numel() == total_s and torch.equal(play[:off_s[6]], blob[:off_a[6]])
    assert torch.equal(_bits(InferencePolicy(play, D)(obs)), _bits(slab.mean[3]))
    snap = it.sim.state_snapshot()
    det = FusedPolicyRollout(it.sim, play, 4, deterministic=True).capture(roll._base).run()
    it.sim.load_state(snap)
    det_a = FusedPolicyRollout(it.sim, blob, 4, deterministic=True).capture(roll._base).run()
    assert torch.equal(_bits(det.actions), _bits(det_a.actions)) and torch.equal(_bits(det.obs), _bits(det_a.obs))
    assert torch.equal(_bits(det.actions[0]), _bits(InferencePolicy(blob, D, critic_obs_dim=29)(det.obs_in[0])))


# ---- the env, the runner and its checkpoints ----------------------------------------------------------------------------------

CRITIC_GROUP = [("pos", "root_pos_w", {}), ("euler", "root_euler_xyz", {}), ("lin", "base_lin_vel", {}), ("ang", "base_ang_vel", {}),
                ("act", "last_action", {"clip": (-1.0, 1.0)})]


def _agent_cfg(activation="elu", save_interval=50, T=24):
    from dataclasses import asdict
    from wheeledlab_b200.learner import PPOConfig
    return {"num_steps_per_env": T, "save_interval": save_interval, "empirical_normalization": False,
            "policy": {"class_name": "ActorCritic", "init_noise_std": 1.0, "actor_hidden_dims": [64, 64], "critic_hidden_dims": [64, 64],
                       "activation": activation},
            "algorithm": {"class_name": "PPO", **asdict(PPOConfig())}}


def _env(n, seed=4, noise=True, critic=None):
    import wheeledlab_b200 as wl
    spec = wl.make_task("Isaac-MushrDriftRL-v0", num_envs=n, seed=seed)
    if not noise:
        for k in range(4):
            spec.cfg.noise_std[k] = 0.0
    env = wl.ManagerBasedRLEnv(spec, device=DEV)
    if critic:
        env.set_critic_observation(critic)
    return env


def test_env_puts_the_critic_group_beside_the_policy_group():
    _need_gpu()
    from wheeledlab_b200 import privileged
    env = _env(64)
    obs, extras = env.reset()
    assert "observations" not in extras and set(obs) == {"policy"} and set(env.observation_manager.group_obs_dim) == {"policy"}
    env.set_critic_observation(CRITIC_GROUP + [("mu", privileged.wheel_friction, {}), ("m", privileged.base_mass, {}),
                                               ("kd", privileged.motor_damping, {})])
    assert env.observation_manager.group_obs_dim["critic"] == (23,)
    obs, extras = env.reset()
    seen = [extras["observations"]["critic"]]
    assert torch.equal(_bits(seen[0]), _bits(env.sim.critic_observe())) and obs["critic"] is seen[0]
    for t in range(5):
        obs, rew, term, trunc, extras = env.step(env.sim.synth_actions(t))
        c = extras["observations"]["critic"]
        assert c.shape == (64, 23) and torch.equal(_bits(c), _bits(env.sim.critic_observe()))
        assert extras["observations"]["policy"] is obs["policy"] and all(c.data_ptr() != x.data_ptr() for x in seen), "a fresh tensor"
        want = torch.cat([privileged.wheel_friction(env), privileged.base_mass(env), privileged.motor_damping(env)], dim=1)
        assert torch.equal(_bits(c[:, 14:]), _bits(want)), "the privileged functions restate the kernel's columns"
        seen.append(c)
    pol, ex = env.get_observations()
    assert torch.equal(_bits(ex["observations"]["critic"]), _bits(env.sim.critic_observe())) and ex["observations"]["policy"] is pol
    with pytest.raises(NotImplementedError, match="Python terms"):
        env.add_reward_term("r", lambda e: torch.zeros(64, device=DEV), 1.0)
    with pytest.raises(NotImplementedError, match="lidar"):
        env.set_critic_observation([("lidar", "lidar_ranges", {})])
    with pytest.raises(ValueError):
        env.sim.critic_observe(out=torch.zeros(64, 14, device=DEV))           # a buffer sized for a narrower table
    env.set_critic_observation([])
    assert "critic" not in env.observation_manager.group_obs_dim and "observations" not in env.step(env.sim.synth_actions(9))[4]


def test_runner_refuses_what_the_asymmetric_iteration_does_not_cover(monkeypatch):
    _need_gpu()
    import wheeledlab_b200 as wl
    from wheeledlab_b200.learner import FusedOnPolicyRunner
    env = _env(64, critic=CRITIC_GROUP)
    with pytest.raises(NotImplementedError, match="relu"):
        FusedOnPolicyRunner(env, _agent_cfg("relu"), device=DEV)
    monkeypatch.setenv("WORLD_SIZE", "2")
    with pytest.raises(NotImplementedError, match="data-parallel"):
        FusedOnPolicyRunner(env, _agent_cfg(), device=DEV)
    monkeypatch.delenv("WORLD_SIZE")
    py = _env(64)
    py.add_reward_term("r", lambda e: torch.zeros(64, device=DEV), 1.0)
    with pytest.raises(NotImplementedError, match="Python terms"):
        py.set_critic_observation(CRITIC_GROUP)
    elev = wl.make("Isaac-MushrElevationRL-v0", device=DEV, num_envs=8, seed=1)
    with pytest.raises(wl.WlError, match="Drift family"):
        elev.set_critic_observation(CRITIC_GROUP)
    assert "critic" not in elev.observation_manager.group_obs_dim


def test_asymmetric_runner_is_one_graph_and_on_the_policy_row_equals_the_symmetric_runner():
    _need_gpu()
    from wheeledlab_b200.learner import FusedOnPolicyRunner, PPOIteration
    runs = []
    for critic in (CRITIC_GROUP, None):
        torch.manual_seed(7)                                  # the same nn.Linear draws: Linear(14, 64) for both critics
        r = FusedOnPolicyRunner(_env(512, noise=False, critic=critic), _agent_cfg(), device=DEV)
        logs = []
        r.callback = lambda k, log: logs.append(log)
        g = torch.Generator(device=DEV).manual_seed(5)
        orig = r.it.run
        r.it.run = lambda: orig(torch.randperm(r.it.perm.numel(), device=DEV, generator=g))
        r.learn(3)
        runs.append((r, logs))
    (a, la), (s, ls) = runs
    assert type(a.it) is PPOIteration and a.it.critic_obs_dim == 14 and a.it.graph is not None and a.it.roll.graph is None
    assert a.critic_obs_dim == 14 and s.critic_obs_dim is None
    assert torch.equal(_bits(a.blob), _bits(s.blob)) and torch.equal(_bits(a.alg.m), _bits(s.alg.m))
    assert torch.equal(_bits(a.alg.state), _bits(s.alg.state)) and torch.equal(a.env.sim.groups, s.env.sim.groups)
    # the episode-log rows are fp32 sums over the envs that reset, formed in each step kernel's own order (the act step's quad
    # kernel here, wl_step's 8-envs-per-CTA kernel there): those entries agree to fp32 rounding, everything else exactly
    for x, y in zip(la, ls):
        assert set(x) == set(y)
        for k in x:
            if k.startswith("Episode_"):
                assert x[k] == pytest.approx(y[k], rel=1e-6, abs=1e-9), k
            elif k != "Perf/total_fps":
                assert x[k] == y[k], k


def test_asymmetric_runner_saves_loads_and_resumes_bit_for_bit(tmp_path):
    _need_gpu()
    from wheeledlab_b200 import privileged
    from wheeledlab_b200.learner import FusedOnPolicyRunner
    group = CRITIC_GROUP + [("mu", privileged.wheel_friction, {}), ("m", privileged.base_mass, {}), ("kd", privileged.motor_damping, {})]
    torch.manual_seed(1)
    env = _env(512, critic=group)
    cfg = _agent_cfg(save_interval=1)
    a = FusedOnPolicyRunner(env, cfg, log_dir=str(tmp_path), device=DEV)
    a.learn(2)
    ck = torch.load(tmp_path / "models" / "model_1.pt")
    assert ck["model_state_dict"]["critic.0.weight"].shape == (64, 23) and ck["iter"] == 1
    kept = str(tmp_path / "kept.pt")                           # (the next learn() writes models/model_1.pt again)
    torch.save(ck, kept)
    assert ck["optimizer_state_dict"]["state"][6]["exp_avg"].shape == (64, 23)
    # rsl_rl's ActorCritic(num_actor_obs=14, num_critic_obs=23, 2): the same keys and shapes load, and its critic reproduces the values
    actor, critic, _ = _nets(0, 23)
    mod = torch.nn.ModuleDict({"actor": actor, "critic": critic})
    mod.load_state_dict({k: v for k, v in ck["model_state_dict"].items() if k != "std"})
    b = FusedOnPolicyRunner(env, cfg, device=DEV)
    assert b.load(str(tmp_path / "models" / "model_1.pt")) is None and b.current_learning_iteration == 1
    for x, y in ((a.blob, b.blob), (a.alg.m, b.alg.m), (a.alg.v, b.alg.v)):
        assert torch.equal(_bits(x), _bits(y))
    a.alg.state[0] = cfg["algorithm"]["learning_rate"]          # (a load restarts the adaptive rate from the cfg's, as rsl_rl)
    a.learn(1)
    slab = a.it.roll.slab
    v64 = critic.double()(slab.critic_obs_in[:-1].double()).squeeze(-1)
    assert (slab.values.double() - v64).abs().max().item() <= 1e-5 * max(1.0, v64.abs().max().item())
    b.it.roll.slab, b.it.roll.obs0, b.it.roll.cobs0 = a.it.roll.slab, a.it.roll.obs0, a.it.roll.cobs0
    b.it.perm.copy_(a.it.perm)
    b.it._learn()
    torch.cuda.synchronize()
    for name, x, y in (("blob", a.blob, b.blob), ("m", a.alg.m, b.alg.m), ("v", a.alg.v, b.alg.v), ("history", a.alg.history, b.alg.history)):
        assert torch.equal(_bits(x), _bits(y)), name
    # a checkpoint of another critic width is refused before anything is written; playback on an env without the group
    # loads the actor of the unchanged checkpoint
    sym = FusedOnPolicyRunner(_env(512), cfg, device=DEV)
    before = sym.blob.clone()
    with pytest.raises(ValueError, match="critic.0"):
        sym.load(kept)
    assert torch.equal(before, sym.blob)
    sym.load(kept, load_optimizer=False)
    obs = slab.obs_in[2]
    c = FusedOnPolicyRunner(env, cfg, device=DEV)
    c.load(kept)
    assert torch.equal(_bits(sym.get_inference_policy()(obs)), _bits(c.get_inference_policy()(obs)))
