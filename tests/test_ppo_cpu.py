"""CPU checks of the PPO learner's host side: the rsl_rl state-dict round trip of the act-step blob, the config, and the
argument errors wl_ppo_update reports before it touches a device."""
import ctypes as C

import torch

KEYS = [f"{net}.{k}.{w}" for net in ("actor", "critic") for k in (0, 2, 4) for w in ("weight", "bias")] + ["std"]


def _nets(obs_dim=14, seed=0):
    torch.manual_seed(seed)
    mk = lambda out: torch.nn.Sequential(torch.nn.Linear(obs_dim, 64), torch.nn.ELU(), torch.nn.Linear(64, 64), torch.nn.ELU(),
                                         torch.nn.Linear(64, out))
    return mk(2), mk(1), torch.tensor([0.7, 1.3])


def test_state_dict_round_trip_is_bit_identical():
    from wheeledlab_b200.policy import actor_critic_state_dict, load_actor_critic_state_dict, pack_actor_critic
    for obs_dim in (14, 13, 16, 1):
        actor, critic, std = _nets(obs_dim)
        blob = pack_actor_critic(actor, critic, std, obs_dim, "cpu")
        sd = actor_critic_state_dict(blob, obs_dim)
        assert list(sd) == KEYS
        ref = {f"actor.{k}": v for k, v in actor.state_dict().items()}
        ref.update({f"critic.{k}": v for k, v in critic.state_dict().items()}, std=std)
        for k in KEYS:
            assert sd[k].shape == ref[k].shape and torch.equal(sd[k], ref[k]), k
        again = load_actor_critic_state_dict(sd, obs_dim, device="cpu")
        assert torch.equal(again.view(torch.int32), blob.view(torch.int32))
        out = torch.full_like(blob, 0.0)
        assert load_actor_critic_state_dict(sd, obs_dim, out=out) is out and torch.equal(out.view(torch.int32), blob.view(torch.int32))


def test_load_state_dict_rejects_other_shapes():
    import pytest
    from wheeledlab_b200.policy import load_actor_critic_state_dict
    actor, critic, std = _nets(12)
    sd = {f"actor.{k}": v for k, v in actor.state_dict().items()}
    sd.update({f"critic.{k}": v for k, v in critic.state_dict().items()}, std=std)
    with pytest.raises(ValueError, match="actor.0"):
        load_actor_critic_state_dict(sd, 14, device="cpu")


def test_ppo_config_defaults_and_from_rsl_rl():
    from types import SimpleNamespace
    from wheeledlab_b200.learner import PPOConfig
    c = PPOConfig()
    assert (c.value_loss_coef, c.use_clipped_value_loss, c.clip_param, c.entropy_coef, c.num_learning_epochs, c.num_mini_batches,
            c.learning_rate, c.schedule, c.gamma, c.lam, c.desired_kl, c.max_grad_norm) == \
        (1.0, True, 0.2, 0.005, 5, 4, 1.0e-3, "adaptive", 0.99, 0.95, 0.01, 1.0)
    alg = SimpleNamespace(class_name="PPO", value_loss_coef=0.5, schedule="fixed", num_mini_batches=8, normalize_advantage_per_mini_batch=False)
    d = PPOConfig.from_rsl_rl(alg)
    assert (d.value_loss_coef, d.schedule, d.num_mini_batches, d.clip_param) == (0.5, "fixed", 8, 0.2)


def test_ppo_update_rejects_bad_arguments_before_any_launch():
    import wheeledlab_b200 as wl
    from wheeledlab_b200._lib import WlPpoBatch, WlPpoParams
    lib = wl.lib
    assert lib.wl_ppo_state_floats() >= 10 + 2 * 20
    fake = 1 << 20                                           # never dereferenced: every call below fails its checks first
    batch = WlPpoBatch(*([fake] * 8))
    params = WlPpoParams(14, 1024, 5, 4, 0.2, 1.0, 0.005, 1.0, 0.01, 1, 1, 0)

    def call(p=params, b=batch, blob=fake):
        rc = lib.wl_ppo_update(C.byref(p) if p is not None else None, C.byref(b) if b is not None else None, blob, fake, fake, fake,
                               fake, 1 << 30, None)
        return rc, lib.wl_last_error().decode()

    rc, msg = call(p=None)
    assert rc == -1 and "wl_ppo_update" in msg and "params" in msg
    rc, msg = call(b=WlPpoBatch(fake, fake, fake, fake, fake, fake, fake, None))
    assert rc == -1 and "wl_ppo_update" in msg and "batch" in msg
    rc, msg = call(blob=None)
    assert rc == -1 and "d_blob" in msg
    rc, msg = call(p=WlPpoParams(17, 1024, 5, 4, 0.2, 1.0, 0.005, 1.0, 0.01, 1, 1, 0))
    assert rc == -3 and "wl_ppo_update" in msg and "obs_dim" in msg
    rc, msg = call(p=WlPpoParams(14, 1022, 5, 4, 0.2, 1.0, 0.005, 1.0, 0.01, 1, 1, 0))
    assert rc == -1 and "wl_ppo_update" in msg and "num_mini_batches" in msg
    assert lib.wl_ppo_workspace_bytes(17, 1024, 4) == 0 and b"wl_ppo_workspace_bytes" in lib.wl_last_error()
