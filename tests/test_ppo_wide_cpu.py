"""CPU checks of the wide (ReLU) learner's host side: the argument errors wl_ppo_update_wide, its workspace query and
wl_policy_act report before they touch a device, and the rsl_rl actor-critic cfg helper."""
import ctypes as C
from types import SimpleNamespace

import pytest


def test_wide_update_rejects_bad_arguments_before_any_launch():
    import wheeledlab_b200 as wl
    from wheeledlab_b200._lib import WlPpoBatch, WlPpoParams
    lib = wl.lib
    fake = 1 << 20                                           # never dereferenced: every call below fails its checks first
    batch = WlPpoBatch(*([fake] * 8))
    params = WlPpoParams(689, 1024, 5, 4, 0.2, 1.0, 0.005, 1.0, 0.01, 1, 1, 0)

    def call(p=params, b=batch, blob=fake):
        rc = lib.wl_ppo_update_wide(C.byref(p) if p is not None else None, C.byref(b) if b is not None else None, blob, fake,
                                    fake, fake, fake, 1 << 30, None)
        return rc, lib.wl_last_error().decode()

    rc, msg = call(p=None)
    assert rc == -1 and "wl_ppo_update_wide" in msg and "params" in msg
    rc, msg = call(b=WlPpoBatch(fake, fake, fake, fake, fake, fake, fake, None))
    assert rc == -1 and "batch" in msg
    rc, msg = call(blob=None)
    assert rc == -1 and "d_blob" in msg
    for D, rc_want in ((0, -1), (4097, -3)):
        rc, msg = call(p=WlPpoParams(D, 1024, 5, 4, 0.2, 1.0, 0.005, 1.0, 0.01, 1, 1, 0))
        assert rc == rc_want and "wl_ppo_update_wide" in msg and "obs_dim" in msg
    rc, msg = call(p=WlPpoParams(689, 1022, 5, 4, 0.2, 1.0, 0.005, 1.0, 0.01, 1, 1, 0))
    assert rc == -1 and "num_mini_batches" in msg
    for D, n, mb in ((0, 1024, 4), (4097, 1024, 4), (689, 1022, 4), (689, 1024, 0)):
        assert lib.wl_ppo_wide_workspace_bytes(D, n, mb) == 0 and b"wl_ppo_wide_workspace_bytes" in lib.wl_last_error()
    # the narrow update still refuses wide observations
    assert lib.wl_ppo_workspace_bytes(689, 1024, 4) == 0


def test_policy_act_rejects_null_arguments():
    import wheeledlab_b200 as wl
    from wheeledlab_b200._lib import WlPolicyOut
    po = WlPolicyOut(1 << 20, 1 << 20, 1 << 20, 1 << 20)
    assert wl.lib.wl_policy_act(None, C.c_void_p(1 << 20), C.c_void_p(1 << 20), po, 0, None) == -1
    assert b"wl_policy_act" in wl.lib.wl_last_error()


def test_activation_from_rsl_rl_policy_cfg():
    from wheeledlab_b200.learner import activation_from_rsl_rl
    cfg = lambda act, a=(64, 64), c=(64, 64): SimpleNamespace(class_name="ActorCritic", init_noise_std=1.0, actor_hidden_dims=list(a),
                                                             critic_hidden_dims=list(c), activation=act)
    assert activation_from_rsl_rl(cfg("relu")) == "relu"
    assert activation_from_rsl_rl(cfg("elu")) == "elu"
    with pytest.raises(NotImplementedError, match="64, 64"):
        activation_from_rsl_rl(cfg("relu", a=(128, 64)))
    with pytest.raises(NotImplementedError):
        activation_from_rsl_rl(cfg("elu", c=(64, 64, 64)))
    with pytest.raises(ValueError, match="tanh"):
        activation_from_rsl_rl(cfg("tanh"))


def test_activation_keyword_is_checked_before_any_device_work():
    import torch
    from wheeledlab_b200.learner import FusedPPO
    from wheeledlab_b200.policy import critic_value
    blob = torch.zeros(16)
    with pytest.raises(ValueError, match="activation"):
        FusedPPO(blob, 1, activation="gelu")
    with pytest.raises(ValueError, match="activation"):
        critic_value(blob, 1, torch.zeros(2, 1), activation="selu")
