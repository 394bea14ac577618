"""The torch restatement of rsl_rl ``PPO.update()`` (tests/ppo_reference.py) for the ReLU actor-critic of the Elevation /
Visual agents (``activation="relu"``): the same TorchPPO with the ELU modules between its layers replaced by ReLU.  The
parameters, the optimiser and the update are TorchPPO's own; only the activation differs."""
from __future__ import annotations

import torch
from torch import nn

from ppo_reference import TorchPPO


def torch_ppo(blob: torch.Tensor, obs_dim: int, cfg, dtype=torch.float32, activation: str = "elu") -> TorchPPO:
    """TorchPPO on the blob's network with `activation` ("elu": unchanged, "relu": both hidden activations of both nets)."""
    if activation not in ("elu", "relu"):
        raise ValueError(f"activation must be 'elu' or 'relu', not {activation!r}")
    r = TorchPPO(blob, obs_dim, cfg, dtype)
    if activation == "relu":
        for net in (r.actor, r.critic):
            for k in (1, 3):
                assert isinstance(net[k], nn.ELU)
                net[k] = nn.ReLU()
    return r
