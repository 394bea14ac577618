"""The learner-facing step right after the rollout (SURVEY 8f-2): returns / advantages over the [T, N] slab.

``compute_returns`` is rsl_rl's ``RolloutStorage.compute_returns`` (called at
``wheeledlab_rl/utils/modified_rsl_rl_runner.py:116``) [UPSTREAM-RECALL], run as one hand-written kernel directly on the
rollout-slab layout (``distributed.RolloutSlab``); advantage normalisation is left to the caller.

``FusedPPO`` is the rest of the iteration, rsl_rl's ``PPO.update()`` (``:118``), on the device (DESIGN 6f).
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass, fields

import torch

from ._lib import WlError, WlPpoBatch, WlPpoParams, check, lib


def compute_returns(rewards: torch.Tensor, values: torch.Tensor, last_values: torch.Tensor, dones: torch.Tensor,
                    gamma: float, lam: float, time_outs: torch.Tensor | None = None):
    """rewards/values [T,N] f32, last_values [N] f32, dones/time_outs [T,N] u8|bool (CUDA, contiguous) -> (returns, advantages)."""
    T, N = rewards.shape
    for x in (rewards, values, last_values, dones):
        if not (x.is_cuda and x.is_contiguous()):
            raise ValueError("compute_returns expects contiguous CUDA tensors")
    d8 = dones.view(torch.uint8) if dones.dtype == torch.bool else dones
    t8 = None if time_outs is None else (time_outs.view(torch.uint8) if time_outs.dtype == torch.bool else time_outs)
    ret, adv = torch.empty_like(rewards), torch.empty_like(rewards)
    stream = C.c_void_p(torch.cuda.current_stream(rewards.device).cuda_stream)
    check(lib.wl_gae(C.c_void_p(rewards.data_ptr()), C.c_void_p(values.data_ptr()), C.c_void_p(last_values.data_ptr()),
                     C.c_void_p(d8.data_ptr()), C.c_void_p(t8.data_ptr()) if t8 is not None else None, gamma, lam,
                     C.c_void_p(ret.data_ptr()), C.c_void_p(adv.data_ptr()), T, N, stream), "wl_gae")
    return ret, adv


class DataParallelAdam:
    """Adam for a (small) set of parameters replicated over the ranks of a process group, with the gradient all-reduce
    fused into the update kernel (``wl_dp_adam_step``): parameters and gradients live in flat buffers (``p.data`` / ``p.grad``
    are views), the flat gradient sits in torch symmetric memory so every rank reads its peers' gradients over NVLink inside
    the update kernel -- one launch per optimiser step, no NCCL call.  world_size 1 (or no process group) is plain fused Adam.
    Matches ``torch.optim.Adam`` (amsgrad off, decoupled weight decay off) on the rank-averaged gradient."""

    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0, group=None):
        import torch.distributed as dist
        self.params = [p for p in params]
        dev = self.params[0].device
        n = sum(p.numel() for p in self.params)
        self.n, self.lr, self.betas, self.eps, self.wd, self.t = n, lr, betas, eps, weight_decay, 0
        self.world = dist.get_world_size(group) if dist.is_initialized() else 1
        self.rank = dist.get_rank(group) if dist.is_initialized() else 0
        self.flat_p = torch.empty(n, dtype=torch.float32, device=dev)
        self.handle = None
        if self.world > 1:
            import torch.distributed._symmetric_memory as symm
            group = group if group is not None else dist.group.WORLD
            self.flat_g = symm.empty(n, dtype=torch.float32, device=dev)
            self.flat_g.zero_()
            self.handle = symm.rendezvous(self.flat_g, group.group_name)
            ptrs = [int(x) for x in self.handle.buffer_ptrs]
        else:
            self.flat_g = torch.zeros(n, dtype=torch.float32, device=dev)
            ptrs = [self.flat_g.data_ptr()]
        self._grad_ptrs = (C.c_void_p * len(ptrs))(*ptrs)
        self.m = torch.zeros(n, dtype=torch.float32, device=dev)
        self.v = torch.zeros(n, dtype=torch.float32, device=dev)
        off = 0
        with torch.no_grad():
            for p in self.params:                          # re-seat parameters and gradients as views of the flat buffers
                k = p.numel()
                self.flat_p[off:off + k].copy_(p.detach().reshape(-1))
                p.data = self.flat_p[off:off + k].view_as(p)
                p.grad = self.flat_g[off:off + k].view_as(p)
                off += k

    def zero_grad(self):
        self.flat_g.zero_()

    def step(self):
        self.t += 1
        stream = C.c_void_p(torch.cuda.current_stream(self.flat_p.device).cuda_stream)
        if self.handle is not None:
            self.handle.barrier()                          # every rank's gradient is complete
        check(lib.wl_dp_adam_step(C.c_void_p(self.flat_p.data_ptr()), C.c_void_p(self.m.data_ptr()), C.c_void_p(self.v.data_ptr()),
                                  self.world, self._grad_ptrs, self.lr, self.betas[0], self.betas[1], self.eps, self.wd, self.t, self.n,
                                  stream), "wl_dp_adam_step")
        if self.handle is not None:
            self.handle.barrier()                          # nobody overwrites a gradient a peer is still reading


@dataclass
class PPOConfig:
    """rsl_rl PPO's algorithm settings [UPSTREAM-RECALL for their meaning].  Defaults are the reference's Drift values,
    ``drifting/config/agents/mushr/rsl_rl_ppo_cfg.py:18-31`` (``MushrPPORunnerCfg.algorithm``); the Adam betas / eps and
    the adaptive-schedule bounds (lr in [1e-5, 1e-2], factor 1.5) are rsl_rl's fixed ones."""
    value_loss_coef: float = 1.0
    use_clipped_value_loss: bool = True
    clip_param: float = 0.2
    entropy_coef: float = 0.005
    num_learning_epochs: int = 5
    num_mini_batches: int = 4
    learning_rate: float = 1.0e-3
    schedule: str = "adaptive"
    gamma: float = 0.99
    lam: float = 0.95
    desired_kl: float = 0.01
    max_grad_norm: float = 1.0

    @classmethod
    def from_rsl_rl(cls, alg_cfg) -> "PPOConfig":
        """The same attribute names read from any object, e.g. the reference's ``RslRlPpoAlgorithmCfg``."""
        return cls(**{f.name: getattr(alg_cfg, f.name) for f in fields(cls) if hasattr(alg_cfg, f.name)})


def activation_from_rsl_rl(policy_cfg) -> str:
    """The hidden activation of an rsl_rl ``RslRlPpoActorCriticCfg``-like object (the reference's ``policy`` of an agent cfg:
    "elu" for the Drift family, "relu" for Elevation and Visual), checked against the network the fused kernels run:
    ``actor_hidden_dims == critic_hidden_dims == [64, 64]`` and ELU or ReLU."""
    from .policy import check_activation
    dims = [list(getattr(policy_cfg, k)) for k in ("actor_hidden_dims", "critic_hidden_dims")]
    if dims != [[64, 64], [64, 64]]:
        raise NotImplementedError(f"the fused actor-critic is [64, 64] for actor and critic, not {dims[0]} / {dims[1]}")
    return check_activation(policy_cfg.activation)


class FusedPPO:
    """rsl_rl ``PPO.update()`` (modified_rsl_rl_runner.py:118) [UPSTREAM-RECALL] on the device, training the blob that
    ``FusedPolicyRollout`` reads in place (``wl_ppo_update``: one gradient kernel + two finisher launches per mini-batch).

    Owns the Adam moments, the device state (learning rate, Adam step, statistics) and the workspace.  Nothing syncs the
    host, so with an explicit ``perm`` tensor refilled in place the update can be captured into the same CUDA graph as the
    rollout.  The network is [64, 64] actor and critic with a learned std: activation "elu" is the Drift family's
    (obs_dim <= 16, ``wl_ppo_update``), "relu" the Elevation / Visual one (obs_dim <= 4096, ``wl_ppo_update_wide``)."""

    def __init__(self, blob: torch.Tensor, obs_dim: int, cfg: PPOConfig | None = None, activation: str = "elu"):
        from .policy import check_activation
        if cfg is None:
            cfg = PPOConfig()
        if cfg.schedule not in ("adaptive", "fixed"):
            raise ValueError(f"schedule must be 'adaptive' or 'fixed', not {cfg.schedule!r}")
        self.blob, self.obs_dim, self.cfg, self.device = blob, obs_dim, cfg, blob.device
        self.activation = check_activation(activation)
        wide = self.activation == "relu"
        self._ws_query = lib.wl_ppo_wide_workspace_bytes if wide else lib.wl_ppo_workspace_bytes
        self._update = lib.wl_ppo_update_wide if wide else lib.wl_ppo_update
        self.m = torch.zeros_like(blob)
        self.v = torch.zeros_like(blob)
        self.state = torch.zeros(lib.wl_ppo_state_floats(), dtype=torch.float32, device=blob.device)
        self.state[0] = cfg.learning_rate
        self.workspace = torch.empty(0, dtype=torch.uint8, device=blob.device)
        self._batch = None

    def _workspace(self, batch: int) -> torch.Tensor:
        with torch.cuda.device(self.device):
            need = self._ws_query(self.obs_dim, batch, self.cfg.num_mini_batches)
        if need == 0:
            raise WlError(f"{self._ws_query.__name__} failed: {lib.wl_last_error().decode()}")
        if self.workspace.numel() < need:
            self.workspace = torch.empty(need, dtype=torch.uint8, device=self.device)
        return self.workspace

    def update(self, slab, returns: torch.Tensor, advantages: torch.Tensor, perm: torch.Tensor | None = None) -> dict:
        """One PPO update over the slab (obs_in / actions / values / log_prob / mean, [T, N, ...]) with returns and
        advantages [T, N] from ``compute_returns``.  perm: int64 [T*N] permutation (default: ``torch.randperm`` on the
        device, as rsl_rl).  Returns device tensors keyed like rsl_rl's loss dict (means over the epochs x mini-batches)
        plus the learning rate and the last mini-batch's KL."""
        cfg = self.cfg
        n = returns.numel()
        if perm is None:
            perm = torch.randperm(n, device=self.device)
        arrays = (slab.obs_in, slab.actions, slab.values, slab.log_prob, slab.mean, returns, advantages, perm)
        for x in arrays:
            if not (x.is_cuda and x.is_contiguous()):
                raise ValueError("FusedPPO.update expects contiguous CUDA tensors")
        if perm.dtype != torch.int64 or perm.numel() != n:
            raise ValueError("perm must be an int64 permutation of the T*N rows")
        ws = self._workspace(n)
        self._batch = WlPpoBatch(*[x.data_ptr() for x in arrays])
        p = WlPpoParams(self.obs_dim, n, cfg.num_learning_epochs, cfg.num_mini_batches, cfg.clip_param, cfg.value_loss_coef,
                        cfg.entropy_coef, cfg.max_grad_norm, cfg.desired_kl, int(cfg.schedule == "adaptive"),
                        int(cfg.use_clipped_value_loss), 0)
        stream = C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)
        check(self._update(C.byref(p), C.byref(self._batch), C.c_void_p(self.blob.data_ptr()), C.c_void_p(self.m.data_ptr()),
                           C.c_void_p(self.v.data_ptr()), C.c_void_p(self.state.data_ptr()), C.c_void_p(ws.data_ptr()),
                           ws.numel(), stream), self._update.__name__)
        k = cfg.num_learning_epochs * cfg.num_mini_batches
        return {"value_function": self.state[7] / k, "surrogate": self.state[6] / k, "entropy": self.state[8] / k,
                "learning_rate": self.state[0], "kl": self.state[9]}

    @property
    def history(self) -> torch.Tensor:
        """[(KL, learning rate used)] per mini-batch of the last update, [epochs * mini-batches, 2] (device view)."""
        k = min(self.cfg.num_learning_epochs * self.cfg.num_mini_batches, (self.state.numel() - 10) // 2)
        return self.state[10:10 + 2 * k].view(k, 2)

    def last_gradient(self) -> torch.Tensor:
        """The last mini-batch's reduced gradient (before clipping), blob layout (device view of the workspace)."""
        return self.workspace[:4 * self.blob.numel()].view(torch.float32)


class PPOIteration:
    """One whole rsl_rl iteration on one GPU (modified_rsl_rl_runner.py:70-118): the fused rollout, the bootstrap value
    V(obs_T) from the blob, ``compute_returns`` (time_outs = truncated, as process_env_step), then ``FusedPPO.update``.
    ``capture=True`` records all of it as ONE CUDA graph; the mini-batch permutation is refilled in place before each
    replay (``torch.randperm`` on the device unless the caller passes one).  ``activation``: as ``FusedPPO``."""

    def __init__(self, sim, blob: torch.Tensor, cfg: PPOConfig | None = None, T: int = 128, activation: str = "elu"):
        from .policy import FusedPolicyRollout
        self.sim, self.blob, self.T = sim, blob, T
        self.roll = FusedPolicyRollout(sim, blob, T, activation=activation)
        self.ppo = FusedPPO(blob, sim.obs_dim, cfg, activation)
        self.perm = torch.empty(T * sim.num_envs, dtype=torch.int64, device=sim.device)
        self.graph = None
        self.stats = None

    def _bootstrap(self) -> torch.Tensor:
        from .policy import critic_value
        return critic_value(self.blob, self.sim.obs_dim, self.roll.obs0, self.ppo.activation)

    def _learn(self):
        slab, cfg = self.roll.slab, self.ppo.cfg
        last_values = self._bootstrap()
        ret, adv = compute_returns(slab.rewards, slab.values, last_values, slab.terminated | slab.truncated, cfg.gamma, cfg.lam,
                                   time_outs=slab.truncated)
        return self.ppo.update(slab, ret, adv, self.perm)

    def start(self, step_counter: int = 0, capture: bool = True):
        roll, sim = self.roll, self.sim
        self.ppo._workspace(self.perm.numel())                 # (allocated outside any capture)
        if not capture:
            roll.capture(step_counter)
            return self
        sim.observe(step_counter, 0, out=roll.obs0)
        sim.set_step_counter(step_counter)
        self.graph = torch.cuda.CUDAGraph()
        s = roll._stream
        s.wait_stream(torch.cuda.current_stream(sim.device))
        with torch.cuda.stream(s):
            self._bootstrap()                                  # warm-up: cuBLAS cannot create its handle under capture
            with torch.cuda.graph(self.graph, stream=s):
                roll._body()
                self.stats = self._learn()
        torch.cuda.current_stream(sim.device).wait_stream(s)
        sim.set_step_counter(step_counter)                     # (the captured advance_counter moved the host mirror)
        roll._base = step_counter
        return self

    def run(self, perm: torch.Tensor | None = None) -> dict:
        self.perm.copy_(perm if perm is not None else torch.randperm(self.perm.numel(), device=self.perm.device))
        if self.graph is None:
            self.roll.run()
            self.stats = self._learn()
            return self.stats
        self.graph.replay()
        self.roll._base += self.T
        self.sim.note_device_counter(self.roll._base)
        return self.stats
