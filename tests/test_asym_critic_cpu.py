"""The asymmetric actor-critic without a GPU (DESIGN 6m): the blob layout with a critic width of its own (host functions of
the library), the rsl_rl state-dict round trip with critic.0.weight [64, Dc], and the refusals that need no device."""
import ctypes as C

import pytest
import torch

D = 14


def _nets(dc, seed=0):
    torch.manual_seed(seed)
    mk = lambda nin, out: torch.nn.Sequential(torch.nn.Linear(nin, 64), torch.nn.ELU(), torch.nn.Linear(64, 64), torch.nn.ELU(),
                                              torch.nn.Linear(64, out))
    return mk(D, 2), mk(dc, 1), torch.tensor([0.7, 1.3])


def test_asym_layout_with_equal_widths_is_the_symmetric_layout():
    from wheeledlab_b200.policy import blob_layout
    for d in range(1, 17):
        assert blob_layout(d, d) == blob_layout(d)


@pytest.mark.parametrize("dc", [1, 3, 14, 17, 29, 32])
def test_asym_layout_sizes_the_critic_first_layer(dc):
    from wheeledlab_b200.policy import blob_layout
    off, total = blob_layout(D, dc)
    sym, _ = blob_layout(D)
    assert off[:7] == sym[:7], "the actor blocks do not move"
    assert off[7] - off[6] == (dc + 3) // 4 * 4 * 64
    assert all(o % 4 == 0 for o in off) and total % 4 == 0 and total == off[12] + 4
    assert [off[k + 1] - off[k] for k in range(7, 12)] == [sym[k + 1] - sym[k] for k in range(7, 12)]


def test_state_dict_round_trip_with_a_critic_width_of_its_own():
    from wheeledlab_b200.policy import actor_critic_state_dict, blob_layout, critic_value, load_actor_critic_state_dict, pack_actor_critic
    dc = 29
    actor, critic, std = _nets(dc)
    blob = pack_actor_critic(actor, critic, std, D, "cpu", critic_obs_dim=dc)
    assert blob.numel() == blob_layout(D, dc)[1]
    sd = actor_critic_state_dict(blob, D, dc)
    assert sd["critic.0.weight"].shape == (64, dc) and sd["actor.0.weight"].shape == (64, D)
    a2, c2, _ = _nets(dc, seed=1)
    torch.nn.ModuleDict({"actor": a2, "critic": c2}).load_state_dict({k: v for k, v in sd.items() if k != "std"})
    x = torch.randn(5, dc)
    assert torch.equal(c2(x), critic(x))
    assert torch.equal(load_actor_critic_state_dict(sd, D, critic_obs_dim=dc), blob)
    assert torch.allclose(critic_value(blob, D, x, critic_obs_dim=dc), critic(x).squeeze(-1), atol=1e-6)
    with pytest.raises(ValueError, match="network shape"):
        pack_actor_critic(actor, critic, std, D, "cpu")            # a [64, 29] critic is not the symmetric network


def test_mismatched_checkpoint_is_refused_with_nothing_written():
    from wheeledlab_b200.policy import actor_critic_state_dict, blob_layout, load_actor_critic_state_dict, pack_actor_critic
    actor, critic, std = _nets(29)
    sd = actor_critic_state_dict(pack_actor_critic(actor, critic, std, D, "cpu", critic_obs_dim=29), D, 29)
    for dc in (None, 17, 32):
        out = torch.full((blob_layout(D, dc)[1],), 7.0)
        with pytest.raises(ValueError, match="critic.0"):
            load_actor_critic_state_dict(sd, D, out=out, critic_obs_dim=dc)
        assert torch.all(out == 7.0), "the actor blocks were written before the critic's shape was checked"


def test_refusals_that_need_no_device():
    from wheeledlab_b200._lib import lib
    from wheeledlab_b200.learner import FusedPPO, PPOConfig
    assert lib.wl_critic_obs_dim(None) == 0
    assert lib.wl_set_critic_terms(None, None, 0) == -1 and b"null handle" in lib.wl_last_error()
    assert lib.wl_critic_observe(None, None, None) == -1
    blob = torch.zeros(16)
    with pytest.raises(NotImplementedError, match="relu"):
        FusedPPO(blob, D, PPOConfig(), activation="relu", critic_obs_dim=20)
    with pytest.raises(NotImplementedError, match="data-parallel"):
        FusedPPO(blob, D, PPOConfig(), exchange=object(), critic_obs_dim=20)


# ---- the critic group of a reference cfg (compat.py, privileged.py) -------------------------------------------------------------

import sys
from pathlib import Path
from types import SimpleNamespace

ROOT = Path(__file__).resolve().parent.parent


@pytest.fixture(scope="module")
def ref_registry():
    if str(ROOT / "shims") not in sys.path:
        sys.path.insert(0, str(ROOT / "shims"))
    import recorded_cfgs
    return recorded_cfgs.load()


def _named(name):
    f = lambda env, **kw: None
    f.__name__ = name
    return f


def _critic_group(**terms):
    from isaaclab.managers import ObservationTermCfg
    g = SimpleNamespace(concatenate_terms=True, enable_corruption=False)
    for k, v in terms.items():
        setattr(g, k, v if hasattr(v, "func") else ObservationTermCfg(func=v))
    return g


def _drift_cfg(reg, gid="Isaac-MushrDriftRL-v0", **terms):
    cfg = reg[gid]["cfgs"]["env_cfg_entry_point"]()
    cfg.scene.num_envs = 16
    if terms:
        cfg.observations.critic = _critic_group(**terms)
    return cfg


def test_compat_lowers_a_critic_group_to_the_term_table(ref_registry):
    from isaaclab.managers import ObservationTermCfg, SceneEntityCfg
    from wheeledlab_b200 import privileged
    from wheeledlab_b200.compat import spec_from_reference_cfg
    pol = _drift_cfg(ref_registry).observations.policy
    terms = {k: ObservationTermCfg(func=t.func, clip=getattr(t, "clip", None))
             for k, t in ((k, getattr(pol, k)) for k in getattr(pol, "_cfg_fields", None) or vars(pol)) if hasattr(t, "func")}
    terms["wheel_spin"] = ObservationTermCfg(func=_named("joint_vel"), params={"asset_cfg": SceneEntityCfg("robot", joint_names=[".*_throttle"])})
    terms["friction"] = privileged.wheel_friction
    terms["mass"] = privileged.base_mass
    terms["damping"] = privileged.motor_damping
    spec = spec_from_reference_cfg(_drift_cfg(ref_registry, **terms))
    assert [(fn, c) for _, fn, c in spec.critic_terms] == [("root_pos_w", 0.0), ("root_euler_xyz", 0.0), ("base_lin_vel", 0.0),
                                                           ("base_ang_vel", 0.0), ("last_action", 1.0), ("joint_vel", 0.0),
                                                           ("wheel_friction", 0.0), ("base_mass", 0.0), ("motor_damping", 0.0)]
    assert privileged.row_width([(fn, c) for _, fn, c in spec.critic_terms]) == 27
    assert spec.critic_terms[5][0] == "wheel_spin"
    # the policy side of the spec is what it is without the group
    plain = spec_from_reference_cfg(_drift_cfg(ref_registry))
    assert plain.critic_terms == [] and bytes(plain.cfg) == bytes(spec.cfg)
    assert (plain.reward_names, plain.termination_names, plain.obs_dim) == (spec.reward_names, spec.termination_names, spec.obs_dim)


def test_compat_refuses_what_the_critic_kernel_does_not_do_by_term_name(ref_registry):
    from isaaclab.managers import ObservationTermCfg, SceneEntityCfg
    from wheeledlab_b200 import privileged
    from wheeledlab_b200.compat import spec_from_reference_cfg
    noise = SimpleNamespace(mean=0.0, std=0.1)
    bad = {
        "noisy_pos": (ObservationTermCfg(func=_named("root_pos_w"), noise=noise), "noise"),
        "scaled_vel": (ObservationTermCfg(func=_named("base_lin_vel"), scale=2.0), "scale"),
        "lidar": (ObservationTermCfg(func=_named("lidar_ranges")), "not in the critic observation library"),
        "lopsided": (ObservationTermCfg(func=_named("last_action"), clip=(-1.0, 2.0)), "symmetric"),
        "steer_rate": (ObservationTermCfg(func=_named("joint_vel"), params={"asset_cfg": SceneEntityCfg("robot", joint_names=[".*_steer"])}),
                       "throttle joints only"),
    }
    for name, (term, msg) in bad.items():
        with pytest.raises(NotImplementedError, match=msg) as e:
            spec_from_reference_cfg(_drift_cfg(ref_registry, **{name: term}))
        assert name in str(e.value)
    cfg = _drift_cfg(ref_registry, friction=privileged.wheel_friction)
    cfg.observations.critic.concatenate_terms = False
    with pytest.raises(NotImplementedError, match="concatenate_terms"):
        spec_from_reference_cfg(cfg)
    wide = {f"spin{k}": _named("joint_vel") for k in range(9)}             # 36 floats
    with pytest.raises(NotImplementedError, match="36 floats") as e:
        spec_from_reference_cfg(_drift_cfg(ref_registry, **wide))
    assert "spin8" in str(e.value)
    for gid, task in (("Isaac-MushrElevationRL-v0", "Elevation"), ("Isaac-MushrVisualRL-v0", "Visual")):
        with pytest.raises(NotImplementedError, match=f"critic observation group on the {task} task"):
            spec_from_reference_cfg(_drift_cfg(ref_registry, gid, friction=privileged.wheel_friction))
    for gid in ("Isaac-F1TenthDriftRL-v0",):
        assert spec_from_reference_cfg(_drift_cfg(ref_registry, gid, mass=privileged.base_mass)).critic_terms == [("mass", "base_mass", 0.0)]


# ---- the asymmetric update restated in fp64 with a hand-written backward pass, against autograd ----------------------------------

def _elu_grad(h):
    return torch.where(h > 0, torch.ones_like(h), h + 1)


def restated_critic_gradients(critic, cobs, values_old, returns, clip, coef):
    """d(coef * clipped value loss)/d(critic parameters) as wl_ppo_grad_asym_kernel forms it: forward over the critic row,
    dV with torch's max / clamp sub-gradients, back-propagation through ELU from the activations, dW1 = cobs^T dz1."""
    (w1, b1), (w2, b2), (w3, b3) = [(critic[k].weight, critic[k].bias) for k in (0, 2, 4)]
    h1 = torch.nn.functional.elu(cobs @ w1.t() + b1)
    h2 = torch.nn.functional.elu(h1 @ w2.t() + b2)
    v = (h2 @ w3.t() + b3).squeeze(-1)
    dvo = v - values_old
    vc = values_old + dvo.clamp(-clip, clip)
    l1, l2 = (v - returns) ** 2, (vc - returns) ** 2
    share = torch.where(l1 > l2, 1.0, torch.where(l1 == l2, 0.5, 0.0)).to(v.dtype)
    inside = ((dvo >= -clip) & (dvo <= clip)).to(v.dtype)
    dv = coef / v.numel() * (share * 2 * (v - returns) + (1 - share) * 2 * (vc - returns) * inside)
    dz2 = (dv[:, None] * w3) * _elu_grad(h2)
    dz1 = (dz2 @ w2) * _elu_grad(h1)
    return {"0.weight": dz1.t() @ cobs, "0.bias": dz1.sum(0), "2.weight": dz2.t() @ h1, "2.bias": dz2.sum(0),
            "4.weight": (dv[:, None] * h2).sum(0, keepdim=True), "4.bias": dv.sum(0, keepdim=True)}


@pytest.mark.parametrize("dc", [17, 29])
def test_fp64_restatement_of_the_asymmetric_critic_gradient_agrees_with_autograd(dc):
    _, critic, _ = _nets(dc, seed=dc)
    critic = critic.double()
    g = torch.Generator().manual_seed(dc)
    n = 2048
    cobs = torch.randn(n, dc, generator=g, dtype=torch.float64)
    with torch.no_grad():
        v0 = critic(cobs).squeeze(-1)
    vo = v0 + 0.25 * torch.randn(n, generator=g, dtype=torch.float64)
    ret = vo + 0.5 * torch.randn(n, generator=g, dtype=torch.float64)
    v = critic(cobs).squeeze(-1)
    vc = vo + (v - vo).clamp(-0.2, 0.2)
    (1.0 * torch.max((v - ret) ** 2, (vc - ret) ** 2).mean()).backward()
    with torch.no_grad():
        got = restated_critic_gradients(critic, cobs, vo, ret, 0.2, 1.0)
    assert got["0.weight"].shape == (64, dc)
    for k, p in critic.named_parameters():
        assert torch.allclose(got[k], p.grad, rtol=1e-9, atol=1e-12), k
