"""The Elevation row critic without a GPU (DESIGN 6s): the lowering of an Elevation ``observations.critic`` group with
``device_terms=True`` and its refusals by term name, the blob layout and rsl_rl state-dict round trip of the wide asymmetric
network at Dc = 689, 690, 701, 721, an fp64 hand-written backward pass of its critic against autograd, and the C ABI's
argument checks that need no device."""
import copy
import sys
from pathlib import Path
from types import SimpleNamespace

import pytest
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
D = 689
ROW = ("goal_relative_xyz", "root_euler_xyz", "base_lin_vel", "base_ang_vel", "last_action", "world_height_map")


@pytest.fixture(scope="module")
def ref_registry():
    if str(ROOT / "shims") not in sys.path:
        sys.path.insert(0, str(ROOT / "shims"))
    import recorded_cfgs
    return recorded_cfgs.load()


def _elev_cfg(reg, gid="Isaac-MushrElevationRL-v0", extra=(), **change):
    """The registered Elevation cfg with a critic group: copies of the policy group's six terms (their functions, params
    and clips), then `extra` (name, ObservationTermCfg); change[name] = {attr: value} edits a row term of the critic."""
    from isaaclab.managers import ObservationTermCfg
    cfg = reg[gid]["cfgs"]["env_cfg_entry_point"]()
    cfg.scene.num_envs = 16
    g = SimpleNamespace(concatenate_terms=True, enable_corruption=False)
    names = []
    for name in vars(cfg.observations.policy):
        t = getattr(cfg.observations.policy, name)
        if hasattr(t, "func"):
            setattr(g, name, ObservationTermCfg(func=t.func, params=dict(t.params or {}), clip=getattr(t, "clip", None)))
            names.append(name)
    for name, attrs in change.items():
        for k, v in attrs.items():
            setattr(getattr(g, name), k, v)
    for name, t in extra:
        setattr(g, name, t)
    cfg.observations.critic = g
    return cfg, names


def _priv():
    from isaaclab.managers import ObservationTermCfg
    from wheeledlab_b200 import privileged
    return [("mu", ObservationTermCfg(func=privileged.wheel_friction)), ("m", ObservationTermCfg(func=privileged.base_mass))]


def test_compat_lowers_an_elevation_critic_group_to_a_row_critic(ref_registry):
    from wheeledlab_b200.compat import spec_from_reference_cfg
    cfg, names = _elev_cfg(ref_registry, extra=_priv(), base_ang_vel={"clip": (-5.0, 5.0)}, elevation_map={"scale": 2.0})
    spec = spec_from_reference_cfg(cfg, device_terms=True)
    assert [fn for _, fn, _ in spec.row_critic] == list(ROW) + ["wheel_friction", "base_mass"]
    assert [n for n, _, _ in spec.row_critic] == names + ["mu", "m"]
    params = [p for _, _, p in spec.row_critic]
    assert params[3] == {"clip": (-5.0, 5.0)} and params[5]["scale"] == 2.0 and params[5]["clip"] == (-10.0, 10.0)
    assert params[0] == {} and params[6] == {} and params[7] == {}
    assert spec.critic_terms == [] and spec.row_terms == []
    with pytest.raises(NotImplementedError, match="Elevation"):
        spec_from_reference_cfg(cfg)                                     # without the flag: today's refusal


def test_compat_refuses_what_the_row_critic_does_not_do_by_term_name(ref_registry):
    from isaaclab.managers import ObservationTermCfg
    from isaaclab.utils.noise import AdditiveGaussianNoiseCfg
    from wheeledlab_b200.compat import spec_from_reference_cfg
    cases = {
        "base_lin_vel": ({"noise": AdditiveGaussianNoiseCfg(std=0.1)}, "noise"),
        "last_action": ({"modifiers": [object()]}, "modifiers"),
        "world_euler_xyz": ({"history_length": 3}, "history_length"),
    }
    for name, (attrs, msg) in cases.items():
        cfg, _ = _elev_cfg(ref_registry, **{name: attrs})
        with pytest.raises(NotImplementedError, match=msg) as e:
            spec_from_reference_cfg(cfg, device_terms=True)
        assert name in str(e.value)
    cfg, _ = _elev_cfg(ref_registry, elevation_map={"scale": tuple([1.0] * 676)})
    with pytest.raises(NotImplementedError, match="per-element scale") as e:
        spec_from_reference_cfg(cfg, device_terms=True)
    assert "elevation_map" in str(e.value)
    cfg, _ = _elev_cfg(ref_registry, elevation_map={"clip": None})
    with pytest.raises(NotImplementedError, match="finite clip") as e:
        spec_from_reference_cfg(cfg, device_terms=True)
    assert "elevation_map" in str(e.value)
    cfg, names = _elev_cfg(ref_registry)                              # row terms out of order
    g = cfg.observations.critic
    a, b = getattr(g, names[2]), getattr(g, names[3])
    setattr(g, names[2], b); setattr(g, names[3], a)
    with pytest.raises(NotImplementedError, match="row order") as e:
        spec_from_reference_cfg(cfg, device_terms=True)
    assert names[2] in str(e.value)
    lidar = lambda env: None
    lidar.__name__ = "lidar_ranges"
    cfg, _ = _elev_cfg(ref_registry, extra=[("lidar", ObservationTermCfg(func=lidar))])
    with pytest.raises(NotImplementedError, match="lidar"):
        spec_from_reference_cfg(cfg, device_terms=True)
    cfg, _ = _elev_cfg(ref_registry)                                  # a library-only group keeps today's refusal
    cfg.observations.critic = SimpleNamespace(concatenate_terms=True, enable_corruption=False, mu=_priv()[0][1])
    with pytest.raises(NotImplementedError, match="Elevation"):
        spec_from_reference_cfg(cfg, device_terms=True)


def test_compat_refuses_a_visual_critic_group(ref_registry):
    from isaaclab.managers import ObservationTermCfg
    from wheeledlab_b200 import privileged
    from wheeledlab_b200.compat import spec_from_reference_cfg
    cfg = ref_registry["Isaac-MushrVisualRL-v0"]["cfgs"]["env_cfg_entry_point"]()
    cfg.scene.num_envs = 16
    cfg.observations.critic = SimpleNamespace(concatenate_terms=True, enable_corruption=False,
                                              mu=ObservationTermCfg(func=privileged.wheel_friction))
    for flag in (False, True):
        with pytest.raises(NotImplementedError, match="Visual"):
            spec_from_reference_cfg(cfg, device_terms=flag)


def test_env_side_lowering_refuses_noise_and_an_unclipped_map():
    from wheeledlab_b200 import row_terms
    assert row_terms.lower_critic_term("m", "world_height_map", None, (-1.0, 1.0), 2.0) == ("world_height_map", None, (-1.0, 1.0), (2.0,))
    with pytest.raises(NotImplementedError, match="noise"):
        row_terms.lower_critic_term("v", "base_lin_vel", ("gaussian", 0.0, 0.1))
    with pytest.raises(NotImplementedError, match="finite clip"):
        row_terms.lower_critic_term("m", "world_height_map", None, None, 2.0)


# ---- the blob layout and the state dict -------------------------------------------------------------------------------------------
def _nets(dc, seed=0):
    torch.manual_seed(seed)
    mk = lambda nin, out: torch.nn.Sequential(torch.nn.Linear(nin, 64), torch.nn.ReLU(), torch.nn.Linear(64, 64), torch.nn.ReLU(),
                                              torch.nn.Linear(64, out))
    return mk(D, 2), mk(dc, 1), torch.tensor([0.7, 1.3])


@pytest.mark.parametrize("dc", [689, 690, 701, 721])
def test_layout_and_state_dict_round_trip(dc):
    from wheeledlab_b200.policy import actor_critic_state_dict, blob_layout, critic_value, load_actor_critic_state_dict, pack_actor_critic
    off, total = blob_layout(D, dc)
    sym_off, sym_total = blob_layout(D)
    assert off[:7] == sym_off[:7], "the actor blocks and the critic's W1t start sit where the symmetric blob has them"
    assert off[7] - off[6] == ((dc + 3) // 4) * 4 * 64
    assert total - sym_total == (off[7] - off[6]) - (sym_off[7] - sym_off[6])
    actor, critic, std = _nets(dc)
    blob = pack_actor_critic(actor, critic, std, D, "cpu", critic_obs_dim=dc)
    sd = actor_critic_state_dict(blob, D, dc)
    assert sd["critic.0.weight"].shape == (64, dc) and sd["actor.0.weight"].shape == (64, D)
    assert torch.equal(load_actor_critic_state_dict(sd, D, critic_obs_dim=dc), blob)
    x = torch.randn(5, dc)
    assert torch.allclose(critic_value(blob, D, x, "relu", dc), critic(x).squeeze(-1), atol=1e-5)
    pad = torch.ones(total, dtype=torch.bool)
    for o, k in zip(off, [D * 64, 64, 4096, 64, 128, 2, dc * 64, 64, 4096, 64, 64, 1, 2]):
        pad[o:o + k] = False
    assert torch.all(blob[pad] == 0)


def test_fp64_hand_backward_of_the_wide_asymmetric_critic_matches_autograd():
    """The critic side of the update, written out as the kernels form it: dz2 = (dV W3) * relu'(h2) (0 at h == 0),
    dz1 = (dz2 W2) * relu'(h1), dW1 = X^T dz1 over the critic's own rows, in fp64 against autograd on the clipped value loss."""
    dc, n, clip, coef = 721, 257, 0.2, 1.0
    _, critic, _ = _nets(dc, seed=3)
    c = copy.deepcopy(critic).double()
    g = torch.Generator().manual_seed(7)
    x = torch.randn(n, dc, generator=g, dtype=torch.float64)
    vo = torch.randn(n, generator=g, dtype=torch.float64)
    R = torch.randn(n, generator=g, dtype=torch.float64)
    V = c(x).squeeze(-1)
    vc = vo + (V - vo).clamp(-clip, clip)
    loss = coef * torch.max((V - R) ** 2, (vc - R) ** 2).mean()
    loss.backward()
    W1, b1, W2, b2, W3, b3 = (p.detach() for p in c.parameters())
    with torch.no_grad():
        h1 = torch.relu(x @ W1.T + b1)
        h2 = torch.relu(h1 @ W2.T + b2)
        v = (h2 @ W3.T + b3).squeeze(-1)
        l1, l2 = (v - R) ** 2, ((vo + (v - vo).clamp(-clip, clip)) - R) ** 2
        w = (l1 > l2).double() + 0.5 * (l1 == l2).double()
        dvo = v - vo
        inside = ((dvo >= -clip) & (dvo <= clip)).double()
        dv = coef / n * (w * 2 * (v - R) + (1 - w) * 2 * (vo + dvo.clamp(-clip, clip) - R) * inside)
        dz2 = (dv[:, None] * W3) * (h2 > 0).double()
        dz1 = (dz2 @ W2) * (h1 > 0).double()
        hand = {"0.weight": dz1.T @ x, "0.bias": dz1.sum(0), "2.weight": dz2.T @ h1, "2.bias": dz2.sum(0),
                "4.weight": dv[None, :] @ h2, "4.bias": dv.sum(0, keepdim=True)}
    for k, p in c.named_parameters():
        assert torch.allclose(hand[k], p.grad, rtol=1e-10, atol=1e-13), k


def test_c_abi_argument_checks_need_no_device():
    import wheeledlab_b200 as wl
    lib = wl.lib
    assert lib.wl_set_row_critic(None, None, 0, None, 0) < 0 and b"null handle" in lib.wl_last_error()
    assert lib.wl_ppo_wide_asym_workspace_bytes(0, 698, 4096, 4) == 0
    assert lib.wl_ppo_wide_asym_workspace_bytes(D, 698, 4096, 3) == 0
