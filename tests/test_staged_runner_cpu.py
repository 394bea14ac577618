"""Training with host-side Python terms, the parts that need no device: wl_policy_act_elu's argument refusal, policy_act's
activation switch, the runner's refusal of Python observation terms (before it touches the env's device) and the order of
the Python terms' log keys."""
import ctypes as C
from types import SimpleNamespace

import pytest
import torch


def test_policy_act_elu_refuses_a_null_handle_without_a_device():
    import wheeledlab_b200 as wl
    from wheeledlab_b200._lib import WlPolicyOut
    po = WlPolicyOut(1 << 20, 1 << 20, 1 << 20, 1 << 20)
    assert wl.lib.wl_policy_act_elu(None, C.c_void_p(1 << 20), C.c_void_p(1 << 20), po, 0, None) == -1
    assert b"wl_policy_act_elu" in wl.lib.wl_last_error()


def test_policy_act_refuses_an_unknown_activation():
    from wheeledlab_b200.policy import policy_act
    with pytest.raises(ValueError, match="activation must be 'elu'"):
        policy_act(None, None, None, None, None, None, None, 0, activation="tanh")


def test_runner_refuses_python_observation_terms_first():
    from wheeledlab_b200.learner import FusedOnPolicyRunner
    from wheeledlab_b200.runs import agent_cfg
    env = SimpleNamespace(_py_obs=[SimpleNamespace(name="speed")], _py_rewards=[SimpleNamespace(name="r")], _py_terms=[])
    with pytest.raises(NotImplementedError, match="Python observation terms"):
        FusedOnPolicyRunner(env, agent_cfg("elu"), device="cuda:0")


def test_python_log_names_follow_the_staged_steps_order():
    from wheeledlab_b200.env import ManagerBasedRLEnv
    env = SimpleNamespace(_py_rewards=[SimpleNamespace(name="a"), SimpleNamespace(name="b")], _py_terms=[SimpleNamespace(name="c")])
    assert ManagerBasedRLEnv.python_log_names.fget(env) == ["Episode_Reward/a", "Episode_Reward/b", "Episode_Termination/c"]
