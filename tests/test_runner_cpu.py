"""CPU checks of the runner's host side: FusedPPO's optimizer state in torch.optim.Adam's state-dict format, the refusals
of malformed optimizer states and agent cfgs, and the reference's agent cfgs mapped to the runner's settings."""
import json
from pathlib import Path

import pytest
import torch

from ppo_reference import TorchPPO

GOLDEN = Path(__file__).resolve().parent / "golden"
KEYS = [f"{net}.{k}.{w}" for net in ("actor", "critic") for k in (0, 2, 4) for w in ("weight", "bias")] + ["std"]


def _fused(obs_dim=14, seed=0, activation="elu"):
    from wheeledlab_b200.learner import FusedPPO, PPOConfig
    from wheeledlab_b200.policy import pack_actor_critic
    torch.manual_seed(seed)
    act = torch.nn.ELU if activation == "elu" else torch.nn.ReLU
    mk = lambda out: torch.nn.Sequential(torch.nn.Linear(obs_dim, 64), act(), torch.nn.Linear(64, 64), act(), torch.nn.Linear(64, out))
    blob = pack_actor_critic(mk(2), mk(1), torch.tensor([0.7, 1.3]), obs_dim, "cpu")
    return FusedPPO(blob, obs_dim, PPOConfig(), activation), blob


def _torch_adam_state(blob, obs_dim, steps=2):
    """The restatement's torch.optim.Adam after `steps` optimiser steps on an arbitrary loss."""
    from wheeledlab_b200.learner import PPOConfig
    ref = TorchPPO(blob, obs_dim, PPOConfig())
    g = torch.Generator().manual_seed(1)
    for _ in range(steps):
        ref.optimizer.zero_grad()
        x = torch.randn(16, obs_dim, generator=g)
        (ref.actor(x).square().sum() + ref.critic(x).sum() + ref.std.prod()).backward()
        ref.optimizer.step()
    return ref.optimizer.state_dict()


@pytest.mark.parametrize("obs_dim", [14, 689])
def test_optimizer_state_dict_has_torch_adams_structure(obs_dim):
    ppo, blob = _fused(obs_dim, activation="elu" if obs_dim <= 16 else "relu")
    want = _torch_adam_state(blob, obs_dim)
    assert ppo.optimizer_state_dict() == {"state": {}, "param_groups": [{**want["param_groups"][0], "lr": pytest.approx(1e-3)}]}
    ppo.m.copy_(torch.randn_like(ppo.m)); ppo.v.copy_(torch.rand_like(ppo.v)); ppo.state[1] = 2
    got = ppo.optimizer_state_dict()
    assert set(got) == {"state", "param_groups"}
    assert list(got["state"]) == list(want["state"]) == list(range(13))
    assert got["param_groups"][0].keys() == want["param_groups"][0].keys()
    assert got["param_groups"][0]["params"] == want["param_groups"][0]["params"] == list(range(13))
    for k in ("betas", "eps", "weight_decay", "amsgrad"):
        assert got["param_groups"][0][k] == want["param_groups"][0][k]
    for i in range(13):
        assert list(got["state"][i]) == list(want["state"][i]) == ["step", "exp_avg", "exp_avg_sq"]
        assert got["state"][i]["step"].dtype == want["state"][i]["step"].dtype and float(got["state"][i]["step"]) == 2.0
        for k in ("exp_avg", "exp_avg_sq"):
            assert got["state"][i][k].shape == want["state"][i][k].shape, (i, k)


def test_optimizer_state_round_trip_is_bit_identical_and_keeps_padding_zero():
    from wheeledlab_b200.policy import actor_critic_state_dict, load_actor_critic_state_dict
    for obs_dim, act in ((14, "elu"), (13, "elu"), (1, "elu"), (689, "relu")):
        src, blob = _fused(obs_dim, activation=act)
        marker = torch.arange(blob.numel(), dtype=torch.float32) + 1
        touched = torch.zeros_like(blob)
        load_actor_critic_state_dict(actor_critic_state_dict(marker, obs_dim), obs_dim, out=touched)
        pad = touched == 0                                           # blob entries that no parameter maps to
        src.m.copy_(torch.randn_like(src.m).masked_fill(pad, 0.0)); src.v.copy_(torch.rand_like(src.v).masked_fill(pad, 0.0)); src.state[1] = 37
        sd = src.optimizer_state_dict()
        dst, _ = _fused(obs_dim, seed=1, activation=act)
        dst.m.fill_(5.0); dst.v.fill_(5.0); dst.state[0] = 0.25
        dst.load_optimizer_state_dict(sd)
        assert torch.equal(dst.m.view(torch.int32), src.m.view(torch.int32)) and torch.equal(dst.v.view(torch.int32), src.v.view(torch.int32))
        assert (dst.m[pad] == 0).all() and (dst.v[pad] == 0).all()
        assert float(dst.state[1]) == 37.0
        assert float(dst.state[0]) == pytest.approx(1e-3)                 # lr after a load: the cfg's rate, as rsl_rl


def test_torch_adam_state_loads_into_fused_ppo_and_back():
    from wheeledlab_b200.policy import actor_critic_state_dict
    ppo, blob = _fused(14)
    want = _torch_adam_state(blob, 14, steps=3)
    ppo.load_optimizer_state_dict(want)
    assert float(ppo.state[1]) == 3.0
    got = ppo.optimizer_state_dict()
    for i in range(13):
        for k in ("exp_avg", "exp_avg_sq"):
            assert torch.equal(got["state"][i][k], want["state"][i][k]), (i, k)
    names = list(actor_critic_state_dict(blob, 14))
    assert names == KEYS
    # and the fused form loads into torch's Adam
    from wheeledlab_b200.learner import PPOConfig
    ref = TorchPPO(blob, 14, PPOConfig())
    ref.optimizer.load_state_dict(got)
    for i, p in enumerate(ref.parameters()):
        assert torch.equal(ref.optimizer.state[p]["exp_avg"], want["state"][i]["exp_avg"])


def test_malformed_optimizer_states_raise_before_writing():
    ppo, blob = _fused(14)
    good = _torch_adam_state(blob, 14)
    m0 = ppo.m.clone()

    def bad(edit):
        sd = {"state": {i: dict(s) for i, s in good["state"].items()}, "param_groups": [dict(good["param_groups"][0])]}
        edit(sd)
        with pytest.raises(ValueError):
            ppo.load_optimizer_state_dict(sd)
        assert torch.equal(ppo.m, m0)

    bad(lambda sd: sd["state"][0].update(exp_avg=torch.zeros(64, 13)))             # actor.0 of another obs_dim
    bad(lambda sd: sd["state"][12].update(exp_avg_sq=torch.zeros(3)))              # std of three actions
    bad(lambda sd: sd["state"].pop(5))
    bad(lambda sd: sd["state"][4].pop("exp_avg"))
    bad(lambda sd: sd["state"][4].update(step=torch.tensor(9.0)))                  # mixed step counts
    bad(lambda sd: sd["param_groups"][0].update(params=list(range(12))))
    bad(lambda sd: sd["param_groups"][0].update(betas=(0.8, 0.999)))
    bad(lambda sd: sd["param_groups"][0].update(weight_decay=1e-4))
    bad(lambda sd: sd.pop("param_groups"))
    with pytest.raises(ValueError):
        ppo.load_optimizer_state_dict([good])


def _agent_cfgs():
    rec = json.loads((GOLDEN / "rsl_rl_agent_cfgs.json").read_text())
    rec.pop("_source")
    return rec


def test_reference_agent_cfgs_map_to_the_runner_settings():
    from wheeledlab_b200.learner import FusedOnPolicyRunner, PPOConfig
    want_act = {"Isaac-MushrDriftRL-v0": "elu", "Isaac-F1TenthDriftRL-v0": "elu", "Isaac-MushrElevationRL-v0": "relu",
                "Isaac-MushrVisualRL-v0": "relu"}
    cfgs = _agent_cfgs()
    assert set(cfgs) == set(want_act)
    for gid, cfg in cfgs.items():
        s = FusedOnPolicyRunner.settings(cfg)
        assert (s.num_steps_per_env, s.save_interval, s.activation, s.init_noise_std) == (128, 50, want_act[gid], 1.0), gid
        assert s.alg_cfg == PPOConfig(), gid                                            # every agent cfg uses rsl_rl's Drift values


def test_runner_refuses_what_it_cannot_run():
    from wheeledlab_b200.learner import FusedOnPolicyRunner
    cfg = _agent_cfgs()["Isaac-MushrDriftRL-v0"]
    with pytest.raises(NotImplementedError, match="empirical_normalization"):
        FusedOnPolicyRunner(None, {**cfg, "empirical_normalization": True})
    with pytest.raises(NotImplementedError, match="ActorCriticRecurrent"):
        FusedOnPolicyRunner.settings({**cfg, "policy": {**cfg["policy"], "class_name": "ActorCriticRecurrent"}})
    with pytest.raises(NotImplementedError, match="64, 64"):
        FusedOnPolicyRunner.settings({**cfg, "policy": {**cfg["policy"], "actor_hidden_dims": [256, 128]}})


def test_episode_stats_rejects_bad_arguments_before_any_launch():
    import ctypes as C
    import wheeledlab_b200 as wl
    from wheeledlab_b200._lib import WlEpisodeStatsState
    lib = wl.lib
    assert C.sizeof(WlEpisodeStatsState) == 832 and WlEpisodeStatsState.mean_return.offset == 816
    assert lib.wl_episode_stats_workspace_bytes(128, 4096) >= 8 * 128 * 4096 + 4 * 128 * 128
    for T, N in ((0, 16), (4097, 16), (8, 0)):
        assert lib.wl_episode_stats_workspace_bytes(T, N) == 0 and b"wl_episode_stats_workspace_bytes" in lib.wl_last_error()
    fake = C.c_void_p(1 << 20)
    ok = (fake, fake, fake, 128, 4096, fake, fake, fake, fake, 1 << 30, None)
    assert lib.wl_episode_stats(*ok[:7], None, *ok[8:]) == -1 and b"null" in lib.wl_last_error()
    assert lib.wl_episode_stats(*ok[:3], 5000, *ok[4:]) == -1 and b"T must" in lib.wl_last_error()
    assert lib.wl_episode_stats(*ok[:9], 1024, None) == -1 and b"workspace" in lib.wl_last_error()
    assert lib.wl_episode_stats(*ok[:7], C.c_void_p((1 << 20) + 4), *ok[8:]) == -1 and b"aligned" in lib.wl_last_error()
