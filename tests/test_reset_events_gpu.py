"""Reset-mode domain randomisation on the device (DESIGN 6n): wl_reset_dr_kernel after every call that resets envs, against
the oracle bit for bit, on every step entry point and kernel variant; what it leaves alone; its invariance under sharding
and graph capture; the calls that refuse it."""
import os
import sys
from pathlib import Path
from types import SimpleNamespace

import numpy as np
import pytest
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent))

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
D = 14
ALL = {"material": True, "actuator_gains": True, "base_mass": True}
G_POS, G_PMASS, G_PMU_D, G_PMU_C, G_PKD, G_PIW = 0, 9, 10, 11, 12, 15
DR_GROUPS = [G_PMASS, G_PMU_D, G_PMU_C, G_PKD, G_PIW]


def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")


def _bits(x):
    return x.contiguous().view(torch.int32)


def _sim(task, n, events, seed=3, offset=0, variant=None):
    import wheeledlab_b200 as wl
    spec = wl.make_task(task, num_envs=n, seed=seed, env_id_offset=offset)
    sim = wl.WheeledSim(spec, DEV)
    if variant is not None:
        sim.set_kernel_variant(variant)
    sim.set_reset_events(**events)
    sim.startup()
    sim.reset(None, 0)
    return sim


def _oracle(task, n, mask, seed=3, offset=0):
    from oracle_lib import Oracle
    import wheeledlab_b200 as wl
    spec = wl.make_task(task, num_envs=n, seed=seed, env_id_offset=offset)
    o = Oracle(spec.cfg, heightfield=spec.heightfield, threads=os.cpu_count() or 1)
    assert o.set_reset_events(mask) == 0
    o.startup()
    o.reset(None, 0)
    return o


def _same_state(sim, o, what):
    got = sim.groups.cpu().numpy().view(np.uint32)
    want = o.export_state().view(np.uint32)
    bad = np.argwhere(got != want)
    assert bad.size == 0, f"{what}: {len(bad)} words differ, first (group, env, lane) {bad[:4].tolist()}"


# ---- parity with the oracle -----------------------------------------------------------------------------------------------------

# Elevation is the oracle's expensive task (its height scan, ~0.2 ms per env-step on 8 CPU threads): 256 envs over 300 steps,
# which crosses its 200-step time-out.
@pytest.mark.parametrize("task,n,steps,events", [
    ("drift", 4096, 1000, ALL), ("f1tenth_drift", 1024, 1000, ALL), ("hound_4wd", 8192, 1000, ALL),
    ("elevation", 256, 300, {"material": True, "base_mass": True}),
    ("visual_random", 1024, 1000, {"material": True, "base_mass": True, "wheel_mass": True}),
])
def test_step_redraw_equals_the_oracle(task, n, steps, events):
    _need_gpu()
    variants = [0, 1, 4, 8] if task == "drift" else [0]
    sims = [_sim(task, n, events, variant=v) for v in variants]
    o = _oracle(task, n, sims[0].reset_events)
    _same_state(sims[0], o, f"{task} after startup + reset")
    start = sims[0].groups[DR_GROUPS].clone()
    resets = 0
    for t in range(1, steps + 1):
        a = sims[0].synth_actions(t)
        for s in sims:
            obs, _, term, trunc = s.step(a, t)
        _, _, oterm, otrunc = o.step(a.cpu().numpy(), t)
        resets += int((oterm | otrunc).sum())
        if t % 250 == 0 or t == steps:
            for v, s in zip(variants, sims):
                _same_state(s, o, f"{task} n={n} variant {v} step {t}")
    assert resets > n // 4, "the trajectory crossed too few resets"
    assert not torch.equal(sims[0].groups[DR_GROUPS], start), "the parameters were redrawn"


def test_act_steps_staged_step_and_step_terms_redraw_as_wl_step():
    """The other entry points that reset envs, each against wl_step (and wl_step_terms against the oracle's twin) fed the
    same actions: states equal bit for bit over 600 steps of Drift 4096."""
    _need_gpu()
    from wheeledlab_b200._lib import WlPolicyOut, check, lib
    import ctypes as C
    from wheeledlab_b200.policy import pack_actor_critic
    n, steps = 4096, 600
    torch.manual_seed(1)
    mk = lambda nin, out: torch.nn.Sequential(torch.nn.Linear(nin, 64), torch.nn.ELU(), torch.nn.Linear(64, 64), torch.nn.ELU(),
                                              torch.nn.Linear(64, out)).to(DEV)
    blob = pack_actor_critic(mk(D, 2), mk(D, 1), torch.tensor([0.8, 1.2], device=DEV), D, DEV)
    act, inf, ref_a, ref_i, staged, ref_s, terms = (_sim("drift", n, ALL) for _ in range(7))
    terms.set_device_terms([(1, 0, 0.5, ())])                            # forward_vel, reward role: changes rewards, not the state
    o = _oracle("drift", n, act.reset_events)
    o.set_device_terms([(1, 0, 0.5, ())])
    p = lambda x: C.c_void_p(x.data_ptr())
    obs_a = torch.zeros(n, D, device=DEV)
    obs_a.copy_(act.observe(0))
    obs_i = obs_a.clone()
    outs = [torch.zeros(n, 2, device=DEV), torch.zeros(n, 2, device=DEV), torch.zeros(n, device=DEV), torch.zeros(n, device=DEV)]
    acts_i = torch.zeros(n, 2, device=DEV)
    rew, term, trunc = torch.zeros(n, device=DEV), torch.zeros(n, dtype=torch.uint8, device=DEV), torch.zeros(n, dtype=torch.uint8, device=DEV)
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    for t in range(1, steps + 1):
        nxt = torch.empty_like(obs_a)
        check(lib.wl_act_step(act._h, p(obs_a), p(blob), WlPolicyOut(*(x.data_ptr() for x in outs)), p(nxt), p(rew), p(term), p(trunc),
                              None, t, stream), "wl_act_step")
        ref_a.step(outs[0].clone(), t)
        obs_a = nxt
        nxt = torch.empty_like(obs_i)
        check(lib.wl_act_infer_step(inf._h, p(obs_i), p(blob), p(acts_i), p(nxt), p(rew), p(term), p(trunc), None, t, stream),
              "wl_act_infer_step")
        ref_i.step(acts_i.clone(), t)
        obs_i = nxt
        a = ref_s.synth_actions(t)
        _, bits = staged.step_stage_a(a, t)
        staged.step_stage_b(bits, t)
        ref_s.step(a, t)
        terms.step_terms(a, t)
        o.step_terms(a.cpu().numpy(), t)
    for x, y, name in ((act, ref_a, "wl_act_step"), (inf, ref_i, "wl_act_infer_step"), (staged, ref_s, "staged step")):
        assert torch.equal(x.groups.view(torch.int32), y.groups.view(torch.int32)), name
    _same_state(terms, o, "wl_step_terms")
    assert not torch.equal(ref_s.groups[DR_GROUPS], _sim("drift", n, {}).groups[DR_GROUPS])


# ---- locality ---------------------------------------------------------------------------------------------------------------------

def test_only_the_envs_a_launch_reset_are_redrawn_and_start_up_components_keep_their_bits():
    """Visual random cfg with the base mass in reset mode and the wheel masses in start-up mode, as its own cfg splits them;
    wl_reset with ids redraws exactly those ids."""
    _need_gpu()
    n = 2048
    sim, start = _sim("visual_random", n, {"base_mass": True}), _sim("visual_random", n, {})
    s0 = start.groups.clone()
    prev = sim.groups.clone()
    redrawn = 0
    for t in range(1, 400):
        sim.step(sim.synth_actions(t), t)
        s = sim.groups.clone()
        reset = s[G_POS, :, 3].view(torch.int32) == 0
        for g in DR_GROUPS:
            assert torch.equal(_bits(s[g][~reset]), _bits(prev[g][~reset])), (t, g)
        for g in (G_PMU_D, G_PMU_C, G_PKD, G_PIW):
            assert torch.equal(_bits(s[g]), _bits(s0[g])), (t, g)
        assert bool((s[G_PMASS][reset, 0] != prev[G_PMASS][reset, 0]).all())
        redrawn += int(reset.sum())
        prev = s
    assert redrawn > n
    ids = torch.tensor([5, 6, 2000], dtype=torch.int64, device=DEV)
    sim.reset(ids, 400)
    s = sim.groups.clone()
    keep = torch.ones(n, dtype=torch.bool, device=DEV)
    keep[ids] = False
    assert torch.equal(_bits(s[G_PMASS][keep]), _bits(prev[G_PMASS][keep]))
    assert bool((s[G_PMASS][ids, 0] != prev[G_PMASS][ids, 0]).all())


def test_mask_zero_launches_nothing_new_and_a_mask_one_kernel_per_call():
    _need_gpu()
    n = 1024
    plain, cleared, masked = _sim("drift", n, {}), _sim("drift", n, ALL), _sim("drift", n, ALL)
    cleared.set_reset_events()
    assert plain.reset_events == cleared.reset_events == 0 and masked.reset_events == 7
    sims = (plain, cleared, masked)
    counts = [s.launch_count for s in sims]
    for s in sims:
        s.reset(None, 0)
    assert [s.launch_count - c for s, c in zip(sims, counts)] == [1, 1, 2], "wl_reset: one more launch with the mask"
    counts = [s.launch_count for s in sims]
    for t in range(1, 50):
        for s in sims:
            s.step(s.synth_actions(t), t)
    d = [s.launch_count - c for s, c in zip(sims, counts)]
    assert d[0] == d[1] and d[2] == d[0] + 49


# ---- invariance -------------------------------------------------------------------------------------------------------------------

def test_two_shards_equal_one_handle():
    _need_gpu()
    n = 2048
    whole = _sim("hound_4wd", 2 * n, ALL)
    shards = [_sim("hound_4wd", n, ALL, offset=k * n) for k in range(2)]
    for t in range(1, 600):
        a = whole.synth_actions(t)
        whole.step(a, t)
        for k, s in enumerate(shards):
            s.step(a[k * n:(k + 1) * n].contiguous(), t)
    assert torch.equal(torch.cat([s.groups for s in shards], dim=1).view(torch.int32), whole.groups.view(torch.int32))


def _perms(n, k):
    g = torch.Generator(device=DEV).manual_seed(123)
    return [torch.randperm(n, device=DEV, generator=g) for _ in range(k)]


def test_captured_iteration_equals_eager_and_critic_columns_change_exactly_at_resets():
    _need_gpu()
    from wheeledlab_b200.learner import PPOConfig, PPOIteration
    from wheeledlab_b200.policy import pack_actor_critic
    n, T = 512, 64
    terms = ["root_pos_w", "root_euler_xyz", "base_lin_vel", "base_ang_vel", ("last_action", 1.0), "wheel_friction", "base_mass", "motor_damping"]
    its = []
    for capture in (True, False):
        sim = _sim("drift", n, ALL, seed=2)
        dc = sim.set_critic_terms(terms)
        torch.manual_seed(2)
        mk = lambda nin, out: torch.nn.Sequential(torch.nn.Linear(nin, 64), torch.nn.ELU(), torch.nn.Linear(64, 64), torch.nn.ELU(),
                                                  torch.nn.Linear(64, out)).to(DEV)
        blob = pack_actor_critic(mk(D, 2), mk(dc, 1), torch.ones(2, device=DEV), D, DEV, critic_obs_dim=dc)
        # (started at counter 1: a step at counter 0 redraws with the key of the wl_reset(.., 0) before it, so an env reset
        # there keeps the parameters it was just given)
        its.append((PPOIteration(sim, blob, PPOConfig(), T, episode_stats=True, critic=True).start(1, capture=capture), blob))
    (cap, blob_c), (eag, blob_e) = its
    assert cap.graph is not None and eag.graph is None
    launches = cap.sim.launch_count
    done_any = 0
    for p in _perms(n * T, 5):
        cap.run(p)
        eag.run(p)
        torch.cuda.synchronize()
        slab = cap.roll.slab
        dr = slab.critic_obs_in[:, :, 14:23]                         # friction [4], mass [1], damping [4]
        done = (slab.terminated | slab.truncated).bool()             # [T, N]: step t reset the env
        changed = (dr[1:] != dr[:-1]).any(-1)                        # row t + 1 is formed from the state step t left
        assert torch.equal(changed, done), "the DR columns change exactly at resets"
        done_any += int(done.sum())
    assert done_any > 0
    assert cap.sim.launch_count == launches, "the captured iteration launches nothing outside its graph"
    for a, b, name in ((blob_c, blob_e, "blob"), (cap.sim.groups, eag.sim.groups, "env state"),
                       (cap.roll.slab.flat, eag.roll.slab.flat, "slab"), (cap.ppo.state, eag.ppo.state, "ppo state")):
        assert torch.equal(a.view(torch.uint8), b.view(torch.uint8)), name


def test_runner_applies_the_spec_events_and_trains_inside_its_graph():
    _need_gpu()
    import wheeledlab_b200 as wl
    from wheeledlab_b200.learner import FusedOnPolicyRunner
    spec = wl.make_task("Isaac-MushrDriftRL-v0", num_envs=512, seed=4)
    spec.reset_events = ["material", "actuator_gains", "base_mass"]
    env = wl.ManagerBasedRLEnv(spec, device=DEV)
    assert env.sim.reset_events == 7
    start = env.sim.groups[DR_GROUPS].clone()
    agent = {"num_steps_per_env": 64, "save_interval": 50, "empirical_normalization": False,
             "policy": {"class_name": "ActorCritic", "init_noise_std": 1.0, "actor_hidden_dims": [64, 64], "critic_hidden_dims": [64, 64],
                        "activation": "elu"},
             "algorithm": {"class_name": "PPO"}}
    from dataclasses import asdict
    from wheeledlab_b200.learner import PPOConfig
    agent["algorithm"].update(asdict(PPOConfig()))
    r = FusedOnPolicyRunner(env, agent, device=DEV)
    logs = []
    r.callback = lambda k, log: logs.append(log)
    r.learn(4)
    assert r.it.graph is not None and len(logs) == 4 and sum(x["Episodes/finished"] for x in logs) > 0
    assert env.sim.reset_events == 7 and not torch.equal(env.sim.groups[DR_GROUPS], start)


# ---- refusals ---------------------------------------------------------------------------------------------------------------------

def test_refusals_leave_the_handle_and_its_outputs_untouched():
    _need_gpu()
    import wheeledlab_b200 as wl
    from wheeledlab_b200._lib import lib
    sim = _sim("drift", 256, {"material": True})
    for t in range(1, 20):
        sim.step(sim.synth_actions(t), t)
    before, launches = sim.groups.clone(), sim.launch_count
    assert lib.wl_set_reset_events(sim._h, 16) == -1 and "unknown" in lib.wl_last_error().decode()
    with pytest.raises(wl.WlError, match="wheel-mass"):
        sim.set_reset_events(wheel_mass=True)
    assert sim.reset_events == 1
    K = 4
    slab = SimpleNamespace(actions=torch.full((K, 256, 2), 7.0, device=DEV), obs=torch.full((K, 256, D), 7.0, device=DEV),
                           rewards=torch.full((K, 256), 7.0, device=DEV), terminated=torch.full((K, 256), 7, dtype=torch.uint8, device=DEV),
                           truncated=torch.full((K, 256), 7, dtype=torch.uint8, device=DEV))
    logs = torch.full((K, 16), 7.0, device=DEV)
    with pytest.raises(wl.WlError, match="reset-mode"):
        sim.rollout(K, 20, slab, logs)
    torch.cuda.synchronize()
    assert all(bool((x == 7).all()) for x in (slab.actions, slab.obs, slab.rewards, slab.terminated, slab.truncated, logs))
    assert torch.equal(sim.groups, before) and sim.launch_count == launches
    for task, ev in (("visual", {"material": True}), ("elevation", {"actuator_gains": True})):
        s = wl.WheeledSim(wl.make_task(task, num_envs=8, seed=1), DEV)
        with pytest.raises(wl.WlError, match="wl_set_reset_events"):
            s.set_reset_events(**ev)
        assert s.reset_events == 0
    sim.set_reset_events()
    sim.rollout(K, 20, slab, logs)                                     # mask 0: the rollout runs again
