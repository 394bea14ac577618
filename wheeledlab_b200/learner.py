"""The learner-facing step right after the rollout (SURVEY 8f-2): returns / advantages over the [T, N] slab.

``compute_returns`` is rsl_rl's ``RolloutStorage.compute_returns`` (called at
``wheeledlab_rl/utils/modified_rsl_rl_runner.py:116``) [UPSTREAM-RECALL], run as one hand-written kernel directly on the
rollout-slab layout (``distributed.RolloutSlab``); advantage normalisation is left to the caller.

``FusedPPO`` is the rest of the iteration, rsl_rl's ``PPO.update()`` (``:118``), on the device (DESIGN 6f).

``EpisodeStatistics`` is the runner's episode bookkeeping (``:55-63, :99-109``) and ``FusedOnPolicyRunner`` the runner
itself (``learn`` / ``save`` / ``load`` in rsl_rl's checkpoint format) over ``PPOIteration`` (DESIGN 6h).
"""
from __future__ import annotations

import ctypes as C
import os
import time
from dataclasses import dataclass, fields
from types import SimpleNamespace

import torch

from ._lib import WL_ACTIVATION, WlEpisodeStatsState, WlError, WlPpoBatch, WlPpoParams, check, lib


def compute_returns(rewards: torch.Tensor, values: torch.Tensor, last_values: torch.Tensor, dones: torch.Tensor,
                    gamma: float, lam: float, time_outs: torch.Tensor | None = None):
    """rewards/values [T,N] f32, last_values [N] f32, dones/time_outs [T,N] u8|bool (CUDA, contiguous) -> (returns, advantages).
    Every tensor is checked before the launch (the kernel reads raw pointers: a wrong dtype is misread, a short or host
    tensor is read out of bounds); ``time_outs=None`` is the same as all-zero time-outs."""
    if rewards.dim() != 2:
        raise ValueError(f"compute_returns: rewards must be [T, N], not {tuple(rewards.shape)}")
    T, N = rewards.shape
    named = [("rewards", rewards, (T, N)), ("values", values, (T, N)), ("last_values", last_values, (N,)), ("dones", dones, (T, N))]
    if time_outs is not None:
        named.append(("time_outs", time_outs, (T, N)))
    for name, x, _ in named:
        flag = name in ("dones", "time_outs")
        if flag and x.dtype not in (torch.uint8, torch.bool):
            raise ValueError(f"compute_returns: {name} must be uint8 or bool, not {x.dtype}")
        if not flag and x.dtype != torch.float32:
            raise ValueError(f"compute_returns: {name} must be float32, not {x.dtype}")
    for name, x, shape in named:
        if tuple(x.shape) != shape:
            raise ValueError(f"compute_returns: {name} must have shape {list(shape)}, not {list(x.shape)}")
    for name, x, _ in named:
        if x.device != rewards.device:
            raise ValueError(f"compute_returns: {name} is on {x.device}, rewards on {rewards.device}")
    for name, x, _ in named:
        if not (x.is_cuda and x.is_contiguous()):
            raise ValueError(f"compute_returns: {name} must be a contiguous CUDA tensor")
    d8 = dones.view(torch.uint8) if dones.dtype == torch.bool else dones
    t8 = None if time_outs is None else (time_outs.view(torch.uint8) if time_outs.dtype == torch.bool else time_outs)
    ret, adv = torch.empty_like(rewards), torch.empty_like(rewards)
    stream = C.c_void_p(torch.cuda.current_stream(rewards.device).cuda_stream)
    check(lib.wl_gae(C.c_void_p(rewards.data_ptr()), C.c_void_p(values.data_ptr()), C.c_void_p(last_values.data_ptr()),
                     C.c_void_p(d8.data_ptr()), C.c_void_p(t8.data_ptr()) if t8 is not None else None, gamma, lam,
                     C.c_void_p(ret.data_ptr()), C.c_void_p(adv.data_ptr()), T, N, stream), "wl_gae")
    return ret, adv


class EpisodeStatistics:
    """The runner's episode bookkeeping (modified_rsl_rl_runner.py:55-63, :99-109) on the device: per-env running return
    and length (fp32, as ``cur_reward_sum`` / ``cur_episode_length``) and the last 100 finished episodes (the two
    ``deque(maxlen=100)``), updated once per rollout by ``wl_episode_stats`` without a host sync.  ``state`` may be a
    caller-owned uint8 buffer of ``sizeof(wl_episode_stats_state)`` bytes (8-byte aligned), e.g. part of a read-back block."""

    RING = 100

    def __init__(self, num_envs: int, T: int, device, state: torch.Tensor | None = None):
        self.num_envs, self.T, self.device = num_envs, T, torch.device(device)
        nbytes = C.sizeof(WlEpisodeStatsState)
        if state is None:
            state = torch.zeros(nbytes, dtype=torch.uint8, device=self.device)
        if state.dtype != torch.uint8 or state.numel() != nbytes or state.data_ptr() % 8 or not state.is_cuda:
            raise ValueError(f"state must be {nbytes} contiguous CUDA bytes, 8-byte aligned")
        self.state = state
        f = lambda name: getattr(WlEpisodeStatsState, name).offset
        self.ring_return = state[f("ring_return"):f("ring_length")].view(torch.float32)
        self.ring_length = state[f("ring_length"):f("fill")].view(torch.float32)
        self.counts = state[f("fill"):f("_pad")].view(torch.int32)            # fill, head, finished
        self.means = state[f("mean_return"):nbytes].view(torch.float64)        # mean return, mean length
        self.cur_return = torch.zeros(num_envs, dtype=torch.float32, device=self.device)
        self.cur_length = torch.zeros(num_envs, dtype=torch.float32, device=self.device)
        need = lib.wl_episode_stats_workspace_bytes(T, num_envs)
        if need == 0:
            raise ValueError(lib.wl_last_error().decode())
        self.workspace = torch.empty(need, dtype=torch.uint8, device=self.device)

    def reset(self):
        """Empty the deques and zero the running episodes (the runner's locals at the start of ``learn``), in place."""
        self.state.zero_()
        self.cur_return.zero_()
        self.cur_length.zero_()

    def update(self, rewards: torch.Tensor, terminated: torch.Tensor, truncated: torch.Tensor):
        """rewards [T, N] f32, terminated / truncated [T, N] u8|bool (the rollout slab's fields)."""
        if rewards.dtype != torch.float32:
            raise ValueError(f"EpisodeStatistics.update: rewards must be float32, not {rewards.dtype}")
        for x in (terminated, truncated):
            if x.dtype not in (torch.uint8, torch.bool):
                raise ValueError(f"EpisodeStatistics.update: terminated / truncated must be uint8 or bool, not {x.dtype}")
        for x in (rewards, terminated, truncated):
            if not (x.is_cuda and x.is_contiguous()) or tuple(x.shape) != (self.T, self.num_envs):
                raise ValueError(f"EpisodeStatistics.update expects contiguous [{self.T}, {self.num_envs}] CUDA tensors")
        u8 = lambda x: x.view(torch.uint8) if x.dtype == torch.bool else x
        stream = C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)
        check(lib.wl_episode_stats(C.c_void_p(rewards.data_ptr()), C.c_void_p(u8(terminated).data_ptr()),
                                   C.c_void_p(u8(truncated).data_ptr()), self.T, self.num_envs, C.c_void_p(self.cur_return.data_ptr()),
                                   C.c_void_p(self.cur_length.data_ptr()), C.c_void_p(self.state.data_ptr()),
                                   C.c_void_p(self.workspace.data_ptr()), self.workspace.numel(), stream), "wl_episode_stats")

    def ring(self):
        """(returns, lengths) of the deques on the host, oldest first, as Python floats (one sync)."""
        st = WlEpisodeStatsState.from_buffer_copy(bytes(self.state.cpu().numpy()))
        order = [(st.head - st.fill + k) % self.RING for k in range(st.fill)]
        return [st.ring_return[s] for s in order], [st.ring_length[s] for s in order]


class DataParallelAdam:
    """Adam for a (small) set of parameters replicated over the ranks of a process group, with the gradient all-reduce
    fused into the update kernel (``wl_dp_adam_step``): parameters and gradients live in flat buffers (``p.data`` / ``p.grad``
    are views), the flat gradient sits in torch symmetric memory so every rank reads its peers' gradients over NVLink inside
    the update kernel -- one launch per optimiser step, no NCCL call.  world_size 1 (or no process group) is plain fused Adam.
    Matches ``torch.optim.Adam`` (amsgrad off, decoupled weight decay off) on the rank-averaged gradient.

    ``Module.zero_grad()`` (``set_to_none=True`` by default) drops the seated views, and the next backward writes a fresh
    ``p.grad``.  ``step()`` notices a gradient that is no longer its view of the flat buffer (another storage or shape),
    copies it into the flat buffer and seats the view again, so the update always uses the gradient ``p.grad`` holds; a
    parameter whose ``p.grad`` is None is refused (``torch.optim.Adam`` would skip it, the fused update cannot)."""

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
        self._grad_views = []
        with torch.no_grad():
            for p in self.params:                          # re-seat parameters and gradients as views of the flat buffers
                k = p.numel()
                self.flat_p[off:off + k].copy_(p.detach().reshape(-1))
                p.data = self.flat_p[off:off + k].view_as(p)
                p.grad = self.flat_g[off:off + k].view_as(p)
                self._grad_views.append(p.grad)
                off += k

    def zero_grad(self):
        self.flat_g.zero_()

    def _gather_detached_grads(self):
        """Copy every gradient that is not (any more) the seated view into the flat buffer and seat the view again."""
        with torch.no_grad():
            for i, (p, view) in enumerate(zip(self.params, self._grad_views)):
                g = p.grad
                if g is None:
                    raise ValueError(f"DataParallelAdam.step: parameter {i} has no gradient (p.grad is None)")
                if g.data_ptr() != view.data_ptr() or g.shape != view.shape:
                    view.copy_(g)
                    p.grad = view

    def step(self):
        self._gather_detached_grads()
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
    (obs_dim <= 16, ``wl_ppo_update``), "relu" the Elevation / Visual one (obs_dim <= 4096, ``wl_ppo_update_wide``).

    With an ``exchange`` (``PPOExchange``) the update is rsl_rl's multi-GPU one (``wl_ppo_update_dp``, DESIGN 6j): this
    replica is rank ``exchange.rank`` of ``exchange.n_ranks``, and the gradient and KL are averaged across the ranks inside
    every mini-batch.  ``update_local_ranks`` runs several replicas of one process together.

    ``critic_obs_dim`` (None: the critic reads the policy row) trains the asymmetric network (``wl_ppo_update_asym``, DESIGN
    6m): the blob is laid out by ``blob_layout(obs_dim, critic_obs_dim)`` and the slab carries ``critic_obs_in``
    [T + 1, N, critic_obs_dim].  "elu" for the Drift family (obs_dim <= 16, critic_obs_dim <= 32); "relu" for the wide
    network (obs_dim > 16: the Elevation row critic, ``wl_ppo_update_wide_asym``, DESIGN 6s, critic_obs_dim <= 4096).
    Not with an exchange (its buffers are sized by one obs_dim)."""

    def __init__(self, blob: torch.Tensor, obs_dim: int, cfg: PPOConfig | None = None, activation: str = "elu",
                 exchange: "PPOExchange | None" = None, critic_obs_dim: int | None = None):
        from .policy import check_activation
        if critic_obs_dim is not None and activation != "elu" and obs_dim <= 16:
            raise NotImplementedError('a critic observation group with activation="relu" is not implemented for the Drift family '
                                      '(obs_dim <= 16: ELU only)')
        if critic_obs_dim is not None and exchange is not None:
            raise NotImplementedError("a critic observation group in a data-parallel world is not implemented "
                                      "(the exchange buffer is sized by one obs_dim)")
        self.critic_obs_dim = critic_obs_dim
        if cfg is None:
            cfg = PPOConfig()
        if cfg.schedule not in ("adaptive", "fixed"):
            raise ValueError(f"schedule must be 'adaptive' or 'fixed', not {cfg.schedule!r}")
        self.blob, self.obs_dim, self.cfg, self.device = blob, obs_dim, cfg, blob.device
        self.exchange = exchange
        self.activation = check_activation(activation)
        wide = self.activation == "relu"
        self._asym_ws = lib.wl_ppo_wide_asym_workspace_bytes if wide else lib.wl_ppo_asym_workspace_bytes
        self._asym_update = lib.wl_ppo_update_wide_asym if wide else lib.wl_ppo_update_asym
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
            if self.critic_obs_dim is not None:
                need = self._asym_ws(self.obs_dim, self.critic_obs_dim, batch, self.cfg.num_mini_batches)
            else:
                need = self._ws_query(self.obs_dim, batch, self.cfg.num_mini_batches)
        if need == 0:
            raise WlError(f"the PPO workspace query failed: {lib.wl_last_error().decode()}")
        if self.workspace.numel() < need:
            self.workspace = torch.empty(need, dtype=torch.uint8, device=self.device)
        return self.workspace

    def _prepare(self, slab, returns: torch.Tensor, advantages: torch.Tensor, perm: torch.Tensor | None):
        """Check the update's tensors, size the workspace, keep the batch struct alive: (params, batch, workspace)."""
        cfg = self.cfg
        n = returns.numel()
        if perm is None:
            perm = torch.randperm(n, device=self.device)
        arrays = (slab.obs_in, slab.actions, slab.values, slab.log_prob, slab.mean, returns, advantages, perm)
        if self.critic_obs_dim is not None:
            cobs = getattr(slab, "critic_obs_in", None)
            if cobs is None or cobs.shape[-1] != self.critic_obs_dim or cobs.shape[0] * cobs.shape[1] < n:
                raise ValueError(f"the slab must carry critic_obs_in [T + 1, N, {self.critic_obs_dim}]")
        for x in arrays + ((slab.critic_obs_in,) if self.critic_obs_dim is not None else ()):
            if not (x.is_cuda and x.is_contiguous()):
                raise ValueError("FusedPPO.update expects contiguous CUDA tensors")
        if perm.dtype != torch.int64 or perm.numel() != n:
            raise ValueError("perm must be an int64 permutation of the T*N rows")
        ws = self._workspace(n)
        self._batch = WlPpoBatch(*[x.data_ptr() for x in arrays])
        p = WlPpoParams(self.obs_dim, n, cfg.num_learning_epochs, cfg.num_mini_batches, cfg.clip_param, cfg.value_loss_coef,
                        cfg.entropy_coef, cfg.max_grad_norm, cfg.desired_kl, int(cfg.schedule == "adaptive"),
                        int(cfg.use_clipped_value_loss), 0)
        return p, self._batch, ws

    def _stats(self) -> dict:
        k = self.cfg.num_learning_epochs * self.cfg.num_mini_batches
        return {"value_function": self.state[7] / k, "surrogate": self.state[6] / k, "entropy": self.state[8] / k,
                "learning_rate": self.state[0], "kl": self.state[9]}

    def update(self, slab, returns: torch.Tensor, advantages: torch.Tensor, perm: torch.Tensor | None = None) -> dict:
        """One PPO update over the slab (obs_in / actions / values / log_prob / mean, [T, N, ...]) with returns and
        advantages [T, N] from ``compute_returns``.  perm: int64 [T*N] permutation (default: ``torch.randperm`` on the
        device, as rsl_rl).  Returns device tensors keyed like rsl_rl's loss dict (means over the epochs x mini-batches)
        plus the learning rate and the last mini-batch's KL (with an exchange: this rank's losses, the ranks' mean KL)."""
        if self.exchange is not None:
            if self.exchange.one_process and self.exchange.n_ranks > 1:
                raise ValueError("FusedPPO.update: the ranks of a one-process exchange update together (update_local_ranks)")
            return update_local_ranks([self], [(slab, returns, advantages, perm)])[0]
        p, batch, ws = self._prepare(slab, returns, advantages, perm)
        stream = C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)
        if self.critic_obs_dim is not None:
            check(self._asym_update(C.byref(p), C.byref(batch), C.c_void_p(slab.critic_obs_in.data_ptr()), self.critic_obs_dim,
                                    C.c_void_p(self.blob.data_ptr()), C.c_void_p(self.m.data_ptr()), C.c_void_p(self.v.data_ptr()),
                                    C.c_void_p(self.state.data_ptr()), C.c_void_p(ws.data_ptr()), ws.numel(), stream),
                  self._asym_update.__name__)
            return self._stats()
        check(self._update(C.byref(p), C.byref(batch), C.c_void_p(self.blob.data_ptr()), C.c_void_p(self.m.data_ptr()),
                           C.c_void_p(self.v.data_ptr()), C.c_void_p(self.state.data_ptr()), C.c_void_p(ws.data_ptr()),
                           ws.numel(), stream), self._update.__name__)
        return self._stats()

    @property
    def history(self) -> torch.Tensor:
        """[(KL, learning rate used)] per mini-batch of the last update, [epochs * mini-batches, 2] (device view)."""
        k = min(self.cfg.num_learning_epochs * self.cfg.num_mini_batches, (self.state.numel() - 10) // 2)
        return self.state[10:10 + 2 * k].view(k, 2)

    def last_gradient(self) -> torch.Tensor:
        """The last mini-batch's reduced gradient (before clipping; with an exchange, the ranks' average), blob layout
        (device view of the workspace)."""
        return self.workspace[:4 * self.blob.numel()].view(torch.float32)

    def optimizer_state_dict(self) -> dict:
        """What ``torch.optim.Adam(actor_critic.parameters()).state_dict()`` holds in rsl_rl's checkpoints
        (``optimizer_state_dict``): params 0..12 in ActorCritic order (actor.0/2/4 weight|bias, critic.0/2/4 weight|bias,
        std), ``state[i] = {step, exp_avg, exp_avg_sq}`` with the moments transposed out of the blob layout as
        ``policy.actor_critic_state_dict`` does for the weights (empty before the first update), and one param group with
        the current learning rate.  Reads the device state (one sync)."""
        from .policy import actor_critic_state_dict
        lr, step = (float(x) for x in self.state[:2].tolist())
        m, v = (actor_critic_state_dict(x, self.obs_dim, self.critic_obs_dim) for x in (self.m, self.v))
        state = {} if step == 0 else {i: {"step": torch.tensor(step), "exp_avg": m[k], "exp_avg_sq": v[k]} for i, k in enumerate(m)}
        return {"state": state, "param_groups": [_adam_param_group(lr)]}

    def load_optimizer_state_dict(self, sd: dict):
        """Inverse of ``optimizer_state_dict`` (also for an rsl_rl / torch checkpoint): writes the Adam moments and step count
        in place, so a captured ``PPOIteration`` graph keeps working; padding entries of the moments stay zero.  Shape or
        structure mismatches raise ``ValueError`` before anything is written.

        The learning rate restarts from ``cfg.learning_rate``, not from the saved param group: rsl_rl keeps the adaptive rate
        in ``PPO.learning_rate``, which its ``load`` does not restore, so the first mini-batch after a resume adapts from the
        cfg value [UPSTREAM-RECALL].  (With the "fixed" schedule the rate never moves, so nothing changes.)"""
        from .policy import load_actor_critic_state_dict, actor_critic_state_dict
        if not isinstance(sd, dict) or not isinstance(sd.get("state"), dict) or not isinstance(sd.get("param_groups"), (list, tuple)):
            raise ValueError("optimizer state dict must have 'state' (dict) and 'param_groups' (list)")
        groups = sd["param_groups"]
        if len(groups) != 1 or list(groups[0].get("params", ())) != list(range(13)):
            raise ValueError("optimizer state dict must have one param group over the 13 ActorCritic parameters 0..12")
        g = groups[0]
        if tuple(g.get("betas", ())) != (0.9, 0.999) or g.get("eps") != 1e-8 or g.get("weight_decay", 0) != 0 or g.get("amsgrad", False):
            raise ValueError("the fused update runs Adam with betas (0.9, 0.999), eps 1e-8, no weight decay, no amsgrad (rsl_rl's)")
        names = list(actor_critic_state_dict(self.m, self.obs_dim, self.critic_obs_dim))
        m = torch.zeros_like(self.m)
        v = torch.zeros_like(self.v)
        step = 0.0
        if sd["state"]:
            st = sd["state"]
            if sorted(st) != list(range(13)):
                raise ValueError(f"optimizer state must cover params 0..12, not {sorted(st)}")
            try:
                steps = {float(st[i]["step"]) for i in range(13)}
                for out, key in ((m, "exp_avg"), (v, "exp_avg_sq")):
                    load_actor_critic_state_dict({k: st[i][key] for i, k in enumerate(names)}, self.obs_dim, out=out,
                                                 critic_obs_dim=self.critic_obs_dim)
            except (KeyError, TypeError, RuntimeError) as e:
                raise ValueError(f"malformed optimizer state: {e!r}") from None
            if len(steps) != 1:
                raise ValueError(f"the 13 parameters have different Adam step counts {sorted(steps)}")
            step = steps.pop()
        self.m.copy_(m)
        self.v.copy_(v)
        self.state[1] = step
        self.state[0] = self.cfg.learning_rate


class PPOExchange:
    """The exchange of a data-parallel PPO update (``wl_ppo_update_dp``, DESIGN 6j): ``n_ranks``, this replica's ``rank`` and
    the ``n_ranks`` exchange buffers in rank order (``ptrs``; ``buffer`` is this rank's own, a uint8 device tensor of
    ``wl_ppo_dp_exchange_bytes(obs_dim)`` bytes).  ``symmetric`` allocates it in torch symmetric memory for one rank per
    process; ``local`` allocates the ranks of one process (one device), for the one-process form."""

    def __init__(self, n_ranks: int, rank: int, ptrs, buffer: torch.Tensor, handle=None, one_process: bool = False):
        if not 0 <= rank < n_ranks or len(ptrs) != n_ranks:
            raise ValueError(f"rank {rank} of {n_ranks} with {len(ptrs)} buffers")
        self.n_ranks, self.rank, self.buffer, self.handle = n_ranks, rank, buffer, handle
        self.one_process = one_process
        self.ptrs = (C.c_void_p * n_ranks)(*ptrs)

    @staticmethod
    def nbytes(obs_dim: int) -> int:
        need = lib.wl_ppo_dp_exchange_bytes(obs_dim)
        if need == 0:
            raise WlError(f"wl_ppo_dp_exchange_bytes failed: {lib.wl_last_error().decode()}")
        return need

    @classmethod
    def symmetric(cls, obs_dim: int, device, group=None) -> "PPOExchange":
        """This rank's exchange over the ranks of `group` (default: the world), every buffer P2P-mapped to every rank."""
        import torch.distributed as dist
        import torch.distributed._symmetric_memory as symm
        group = group if group is not None else dist.group.WORLD
        buf = symm.empty(cls.nbytes(obs_dim), dtype=torch.uint8, device=device)
        buf.zero_()
        handle = symm.rendezvous(buf, group.group_name)
        handle.barrier()                                   # every buffer is zero before any rank publishes into it
        return cls(dist.get_world_size(group), dist.get_rank(group), [int(x) for x in handle.buffer_ptrs], buf, handle)

    @classmethod
    def local(cls, n_ranks: int, obs_dim: int, device) -> list:
        """The exchanges of n_ranks ranks that all live in this process on one device (``update_local_ranks``)."""
        bufs = [torch.zeros(cls.nbytes(obs_dim), dtype=torch.uint8, device=device) for _ in range(n_ranks)]
        ptrs = [b.data_ptr() for b in bufs]
        return [cls(n_ranks, r, ptrs, bufs[r], one_process=True) for r in range(n_ranks)]

    def failed(self) -> bool:
        """Whether a peer wait of this rank timed out (its error word; one sync).  The update then stops stepping."""
        return bool(self.buffer[4:8].view(torch.int32).item())

    def check(self):
        if self.failed():
            raise WlError(f"data-parallel PPO update: rank {self.rank} timed out waiting for its peers' gradients "
                          f"(the parameters were left as they were)")


def update_local_ranks(ppos: list, inputs: list) -> list:
    """One data-parallel update of the replicas ``ppos`` (``FusedPPO`` with exchanges of the same ranks, each its own
    rank) in one call: inputs[l] = (slab, returns, advantages, perm) of ppos[l], as ``FusedPPO.update``.  With every rank
    of the exchange local (``PPOExchange.local``) this is the one-process form: the whole exchange on one device and
    stream.  Returns each replica's statistics."""
    if not ppos or len(ppos) != len(inputs):
        raise ValueError("update_local_ranks: one (slab, returns, advantages, perm) per replica")
    ex0 = ppos[0].exchange
    for q in ppos:
        if q.exchange is None or list(q.exchange.ptrs) != list(ex0.ptrs):
            raise ValueError("update_local_ranks: every replica needs an exchange over the same rank buffers")
        if q.activation != ppos[0].activation or q.cfg != ppos[0].cfg or q.obs_dim != ppos[0].obs_dim:
            raise ValueError("update_local_ranks: the replicas must share the network, obs_dim and PPOConfig")
    if len({q.exchange.rank for q in ppos}) != len(ppos):
        raise ValueError("update_local_ranks: two replicas hold the same rank")
    if ex0.one_process and len(ppos) != ex0.n_ranks:
        raise ValueError(f"update_local_ranks: a one-process exchange updates all {ex0.n_ranks} ranks together, not {len(ppos)}")
    prepared = [q._prepare(*x) for q, x in zip(ppos, inputs)]
    nl = len(ppos)
    vp = lambda xs: (C.c_void_p * nl)(*[x.data_ptr() for x in xs])
    batches = (WlPpoBatch * nl)(*[b for _, b, _ in prepared])
    ranks = (C.c_int32 * nl)(*[q.exchange.rank for q in ppos])
    ws = [w for _, _, w in prepared]
    q0 = ppos[0]
    stream = C.c_void_p(torch.cuda.current_stream(q0.device).cuda_stream)
    check(lib.wl_ppo_update_dp(C.byref(prepared[0][0]), WL_ACTIVATION[q0.activation], ex0.n_ranks, ex0.ptrs, nl, ranks, batches,
                               vp([q.blob for q in ppos]), vp([q.m for q in ppos]), vp([q.v for q in ppos]),
                               vp([q.state for q in ppos]), vp(ws), min(w.numel() for w in ws), stream), "wl_ppo_update_dp")
    return [q._stats() for q in ppos]


def _adam_param_group(lr: float) -> dict:
    """torch.optim.Adam's param group as this torch version writes it, for 13 parameters with rsl_rl's settings."""
    group = torch.optim.Adam([torch.zeros(1, requires_grad=True) for _ in range(13)], lr=lr).state_dict()["param_groups"][0]
    group["lr"] = lr
    return group


class PPOIteration:
    """One whole rsl_rl iteration on one GPU (modified_rsl_rl_runner.py:70-118): the fused rollout, the bootstrap value
    V(obs_T) from the blob, ``compute_returns`` (time_outs = truncated, as process_env_step), then ``FusedPPO.update``.
    ``capture=True`` records all of it as ONE CUDA graph; the mini-batch permutation is refilled in place before each
    replay (``torch.randperm`` on the device unless the caller passes one).  ``activation``: as ``FusedPPO``.

    ``episode_stats=True`` adds the runner's episode bookkeeping right after the rollout (``self.episodes``, an
    ``EpisodeStatistics``) and gathers everything the runner logs into one device block, ``self.readback``: the episode
    statistics' state, the update's statistics (``SUMMARY``) and the rollout's T episode-log rows (``roll.logs`` is a view of
    it), so that one copy reads an iteration back.

    ``critic=True`` (a handle with a critic table, ``sim.set_critic_terms``) runs the asymmetric iteration, still one graph:
    the rollout with ``critic=True``, the bootstrap value from the critic row ``critic_obs_in[T]``, and
    ``wl_ppo_update_asym``; the blob is laid out by ``blob_layout(obs_dim, sim.critic_obs_dim)``.  With "relu" (an Elevation
    handle with a row critic, ``sim.set_row_critic``, DESIGN 6s) the update is ``wl_ppo_update_wide_asym``."""

    SUMMARY = ("Loss/value_function", "Loss/surrogate", "Loss/entropy", "Loss/learning_rate", "Policy/mean_noise_std")

    def __init__(self, sim, blob: torch.Tensor, cfg: PPOConfig | None = None, T: int = 128, activation: str = "elu",
                 episode_stats: bool = False, exchange: PPOExchange | None = None, rollout=None, extra_readback_bytes: int = 0,
                 critic: bool = False):
        from .policy import FusedPolicyRollout
        self.sim, self.blob, self.T = sim, blob, T
        self.critic_obs_dim = sim.critic_obs_dim if critic else None
        if critic and rollout is not None:
            raise NotImplementedError("a critic observation group with a caller's rollout (device terms, Python terms) is not implemented")
        self.roll = rollout if rollout is not None else FusedPolicyRollout(sim, blob, T, activation=activation, critic=critic)
        self.ppo = FusedPPO(blob, sim.policy_width, cfg, activation, exchange=exchange, critic_obs_dim=self.critic_obs_dim)
        self.perm = torch.empty(T * sim.num_envs, dtype=torch.int64, device=sim.device)
        self.graph = None
        self.stats = None
        self.episodes = self.readback = self.summary = self.readback_extra = None
        if episode_stats:
            ns = C.sizeof(WlEpisodeStatsState)
            end_logs = ns + 4 * len(self.SUMMARY) + 4 * 16 * T
            extra_at = (end_logs + 7) & ~7
            self.readback = torch.zeros(extra_at + extra_readback_bytes if extra_readback_bytes else end_logs, dtype=torch.uint8,
                                        device=sim.device)
            self.episodes = EpisodeStatistics(sim.num_envs, T, sim.device, state=self.readback[:ns])
            self.summary = self.readback[ns:ns + 4 * len(self.SUMMARY)].view(torch.float32)
            self.roll.logs = self.readback[ns + 4 * len(self.SUMMARY):end_logs].view(torch.float32).view(T, 16)
            if extra_readback_bytes:
                self.readback_extra = self.readback[extra_at:]          # (8-byte aligned)

    def _bootstrap(self) -> torch.Tensor:
        from .policy import critic_value
        if self.critic_obs_dim is not None:                    # cobs0 = critic_obs_in[T] once the rollout has run
            return critic_value(self.blob, self.sim.policy_width, self.roll.cobs0, self.ppo.activation, self.critic_obs_dim)
        return critic_value(self.blob, self.sim.policy_width, self.roll.obs0, self.ppo.activation)

    def _returns(self):
        slab, cfg = self.roll.slab, self.ppo.cfg
        if self.episodes is not None:
            self.episodes.update(slab.rewards, slab.terminated, slab.truncated)
        last_values = self._bootstrap()
        return compute_returns(slab.rewards, slab.values, last_values, slab.terminated | slab.truncated, cfg.gamma, cfg.lam,
                               time_outs=slab.truncated)

    def _learn(self):
        ret, adv = self._returns()
        return self._summarise(self.ppo.update(self.roll.slab, ret, adv, self.perm))

    def _summarise(self, stats):
        if self.summary is not None:
            from .policy import blob_layout
            o_std = blob_layout(self.sim.policy_width, self.critic_obs_dim)[0][12]
            self.summary.copy_(torch.stack([stats["value_function"], stats["surrogate"], stats["entropy"], stats["learning_rate"],
                                            self.blob[o_std:o_std + 2].mean()]))
        return stats

    def start(self, step_counter: int = 0, capture: bool = True):
        roll, sim = self.roll, self.sim
        self.ppo._workspace(self.perm.numel())                 # (allocated outside any capture)
        if not capture:
            roll.capture(step_counter)
            return self
        roll.observe0(step_counter)
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


def device_terms_iteration(env, blob: torch.Tensor, cfg: PPOConfig | None = None, T: int = 128, activation: str = "elu",
                           exchange: PPOExchange | None = None) -> PPOIteration:
    """``PPOIteration`` (episode statistics on) for an env with device terms (``env.add_device_reward_term``): the rollout
    is T x (``policy_act``, ``wl_step_terms``) on device counters, captured in the same graph as the episode statistics,
    bootstrap, GAE and the update; ``exchange`` makes it one rank of a data-parallel run.  The read-back block carries the
    rollout's ``term_logs`` [T, 8] f32 after the episode-log rows."""
    from .policy import FusedPolicyRollout
    sim = env.sim
    roll = FusedPolicyRollout(sim, blob, T, activation=activation, device_terms=True)
    it = PPOIteration(sim, blob, cfg, T, activation, episode_stats=True, exchange=exchange, rollout=roll, extra_readback_bytes=4 * 8 * T)
    roll.term_logs = it.readback_extra.view(torch.float32).view(T, 8)
    return it


class StagedPPOIteration(PPOIteration):
    """``PPOIteration`` for an env with host-side Python reward / termination terms, on one GPU: the rollout is
    ``policy.StagedPolicyRollout`` (T x (policy, ``env.staged_step``), eager: the terms are arbitrary torch code), and
    everything after it -- ``wl_episode_stats``, bootstrap value, GAE, the update and the summary copy, the code
    ``PPOIteration`` captures -- is ONE CUDA graph (``capture=True``).  The read-back block also carries the rollout's
    ``py_logs`` (the Python terms' per-step log entries, f64 [T, len(py_names)]) after the episode-log rows.  The env's
    ``common_step_counter`` advances by T during ``run``."""

    def __init__(self, env, blob: torch.Tensor, cfg: PPOConfig | None = None, T: int = 128, activation: str = "elu"):
        from .policy import StagedPolicyRollout
        roll = StagedPolicyRollout(env, blob, T, activation)
        n_py = len(roll.py_names)
        super().__init__(env.sim, blob, cfg, T, activation, episode_stats=True, rollout=roll, extra_readback_bytes=8 * T * n_py)
        if n_py:
            roll.py_logs = self.readback_extra.view(torch.float64).view(T, n_py)

    def start(self, step_counter: int = 0, capture: bool = True):
        roll, dev = self.roll, self.sim.device
        self.ppo._workspace(self.perm.numel())                 # (allocated outside any capture)
        roll.start(step_counter)
        if capture:
            self.graph = torch.cuda.CUDAGraph()
            s = roll._stream
            s.wait_stream(torch.cuda.current_stream(dev))
            with torch.cuda.stream(s):
                self._bootstrap()                              # warm-up: cuBLAS cannot create its handle under capture
                with torch.cuda.graph(self.graph, stream=s):
                    self.stats = self._learn()
            torch.cuda.current_stream(dev).wait_stream(s)
        return self

    def run(self, perm: torch.Tensor | None = None) -> dict:
        self.perm.copy_(perm if perm is not None else torch.randperm(self.perm.numel(), device=self.perm.device))
        self.roll.run()
        if self.graph is None:
            self.stats = self._learn()
        else:
            self.graph.replay()
        return self.stats


class LocalRanksIteration:
    """The one-process form of a data-parallel iteration: R ``PPOIteration`` s of this process (each with its own sim, blob
    and an exchange from ``PPOExchange.local``) run as one -- every rollout, then every bootstrap and GAE, then one
    ``update_local_ranks`` -- and ``capture=True`` records all of it as ONE CUDA graph.  ``run(perms)`` takes one
    permutation per rank (default: ``torch.randperm`` each)."""

    def __init__(self, its: list):
        if not its or any(it.ppo.exchange is None for it in its):
            raise ValueError("LocalRanksIteration: every iteration needs an exchange")
        self.its, self.graph, self.stats = its, None, None

    def _learn(self):
        inputs = [(it.roll.slab, *it._returns(), it.perm) for it in self.its]
        stats = update_local_ranks([it.ppo for it in self.its], inputs)
        return [it._summarise(st) for it, st in zip(self.its, stats)]

    def _body(self):
        for it in self.its:
            it.roll._body()
        return self._learn()

    def start(self, step_counter: int = 0, capture: bool = True):
        its = self.its
        dev = its[0].sim.device
        for it in its:
            it.ppo._workspace(it.perm.numel())
        if not capture:
            for it in its:
                it.roll.capture(step_counter)
            return self
        for it in its:
            it.roll.observe0(step_counter)
            it.sim.set_step_counter(step_counter)
        self.graph = torch.cuda.CUDAGraph()
        s = its[0].roll._stream
        s.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(s):
            for it in its:
                it._bootstrap()                            # warm-up: cuBLAS cannot create its handle under capture
            with torch.cuda.graph(self.graph, stream=s):
                self.stats = self._body()
        torch.cuda.current_stream(dev).wait_stream(s)
        for it in its:
            it.sim.set_step_counter(step_counter)
            it.roll._base = step_counter
        return self

    def run(self, perms=None) -> list:
        for k, it in enumerate(self.its):
            it.perm.copy_(perms[k] if perms is not None else torch.randperm(it.perm.numel(), device=it.perm.device))
        if self.graph is None:
            for it in self.its:
                it.roll.run()
            self.stats = self._learn()
            return self.stats
        self.graph.replay()
        for it in self.its:
            it.roll._base += it.T
            it.sim.note_device_counter(it.roll._base)
        return self.stats


def _world_size() -> int:
    """The runner's world size, without initialising anything: the process group's, else ``WORLD_SIZE`` (default 1)."""
    import torch.distributed as dist
    return dist.get_world_size() if dist.is_initialized() else int(os.environ.get("WORLD_SIZE", "1"))


def _data_parallel_world(sim, device) -> tuple:
    """(world size, rank) of the runner: (1, 0) without a process group or ``WORLD_SIZE`` > 1; otherwise the process group's
    (initialised here with NCCL if ``WORLD_SIZE`` > 1 asks for one, as rsl_rl does [UPSTREAM-RECALL]) after the checks that
    keep the ranks apart: this rank on ``cuda:LOCAL_RANK``, its env shard at ``env_id_offset = rank * num_envs`` (else the
    ranks would simulate the same envs), no two ranks on one GPU (a peer wait could stall behind the other process)."""
    import torch.distributed as dist
    world = _world_size()
    rank = dist.get_rank() if dist.is_initialized() else int(os.environ.get("RANK", "0"))
    if world <= 1:
        return 1, 0
    if world > 8:
        raise NotImplementedError(f"the data-parallel update exchanges over at most 8 ranks (one node), not {world}")
    local = int(os.environ.get("LOCAL_RANK", rank))
    if torch.device(device) != torch.device(f"cuda:{local}"):
        raise ValueError(f"rank {rank} runs on {device}, not cuda:{local} (LOCAL_RANK): one GPU per rank")
    offset = int(sim.cfg.env_id_offset)
    if offset != rank * sim.num_envs:
        raise ValueError(f"rank {rank}'s env shard starts at env_id_offset {offset}, not rank * num_envs = {rank * sim.num_envs}: "
                         "the ranks would simulate the same envs")
    if not dist.is_initialized():
        torch.cuda.set_device(torch.device(device))
        dist.init_process_group(backend="nccl")
    uuids = [None] * world
    dist.all_gather_object(uuids, str(torch.cuda.get_device_properties(torch.device(device)).uuid))
    if len(set(uuids)) != world:
        raise ValueError(f"two ranks share a GPU (device UUIDs {uuids}): one GPU per rank")
    return world, rank


class FusedOnPolicyRunner:
    """rsl_rl's ``OnPolicyRunner`` as the reference drives it (``modified_rsl_rl_runner.py``, ``train_rl.py:95-116``), over
    ``PPOIteration``: ``FusedOnPolicyRunner(env, agent_cfg.to_dict(), log_dir, device)``, ``learn(n)``, ``save`` / ``load``
    in rsl_rl's checkpoint format.  ``env`` is a ``wheeledlab_b200.env.ManagerBasedRLEnv`` (or a wrapper whose ``unwrapped``
    is one).  Each iteration is ONE CUDA graph -- rollout, ``wl_episode_stats``, bootstrap value, GAE, PPO update -- plus
    the flush of the last episode-log row, and ONE read-back of what is logged.

    An env with host-side Python reward, termination or event terms (``add_reward_term`` / ``add_termination_term`` /
    ``add_event_term``) trains on one GPU through ``StagedPPOIteration``: the rollout runs eagerly, T x (policy, staged step with the terms in between), and
    the rest of the iteration is the same graph; the log gains ``Episode_Reward/<name>`` / ``Episode_Termination/<name>``
    for each Python term, the T-step mean of what env.step's ``extras["log"]`` holds for it.  Python observation terms and
    data-parallel runs with Python terms raise ``NotImplementedError``.  An env with device terms (``add_device_reward_term``)
    trains through ``device_terms_iteration``: its rollout (``policy_act`` then ``wl_step_terms``) is part of the one graph,
    on one GPU or data-parallel, and the log gains each device term's ``Episode_*`` key as its T-step mean.  An env with
    device event terms (``add_device_event_term``) trains the same way; they add no log keys.

    The agent cfg dict is read for ``num_steps_per_env``, ``save_interval``, ``policy`` (``activation_from_rsl_rl``,
    ``init_noise_std``) and ``algorithm`` (``PPOConfig.from_rsl_rl``).  The weights start as the reference's do: torch
    ``nn.Linear`` defaults from torch's global generator, std = ``init_noise_std``.  No writer: ``callback(it, scalars)``,
    if set, receives each iteration's scalars (also kept in ``self.last_log``).

    Data-parallel as rsl_rl [UPSTREAM-RECALL] when ``torch.distributed`` is initialised with a world larger than 1 (or, not
    initialised, when ``WORLD_SIZE`` > 1: the runner then initialises NCCL itself), one process per GPU under ``torchrun``:
    each rank rolls out its own env shard (``env_id_offset = rank * num_envs``), the PPO update averages gradient and KL
    across the ranks inside every mini-batch (``FusedPPO`` with a ``PPOExchange`` in symmetric memory), ``learn`` first
    broadcasts rank 0's weights, only rank 0 saves checkpoints and calls ``callback``, and ``Perf/total_fps`` counts the
    env-steps of every rank.  Every rank loads the same checkpoint.

    An env with a ``critic`` observation group (``env.set_critic_observation``, or a reference cfg with
    ``observations.critic``) trains the asymmetric network (DESIGN 6m): the critic is ``Linear(Dc, 64)``-first and reads the
    critic row, the iteration is ``PPOIteration(critic=True)`` -- still one graph -- and checkpoints keep rsl_rl's keys with
    ``critic.0.weight`` ``[64, Dc]``, as ``ActorCritic(num_actor_obs, num_critic_obs, ...)`` has it.  On one GPU: the ELU
    network on the Drift family, the ReLU network on Elevation with a row critic (DESIGN 6s, noisy row terms included); with
    Python terms, device terms, ``activation="relu"`` on the Drift family or a data-parallel world it raises
    ``NotImplementedError``.

    An env with a policy observation table (``env.set_policy_observation``, or a reference cfg whose ``observations.policy``
    was lowered with ``device_terms=True``; DESIGN 6q) trains its policy on the table's row: the actor (and, without a critic
    group, the critic) is ``Linear(Dp, 64)``-first, the rollout runs the policy kernel on the slab row, the step, then
    ``wl_policy_observe`` into the next slab row, one graph, with device terms, a critic group or data-parallel, and
    checkpoints keep rsl_rl's keys with ``actor.0.weight`` ``[64, Dp]``."""

    @staticmethod
    def settings(train_cfg) -> SimpleNamespace:
        """What the runner reads from an rsl_rl agent cfg (``to_dict()`` form, or the object): num_steps_per_env,
        save_interval, activation, init_noise_std and the PPOConfig.  Raises NotImplementedError for what it cannot run."""
        cfg = train_cfg.to_dict() if hasattr(train_cfg, "to_dict") else dict(train_cfg)
        if cfg.get("empirical_normalization", False):
            raise NotImplementedError("empirical_normalization=True: the fused policy reads raw observations (every reference "
                                      "agent cfg sets it to False)")
        pol, alg = dict(cfg["policy"]), dict(cfg["algorithm"])
        if pol.get("class_name", "ActorCritic") != "ActorCritic" or alg.get("class_name", "PPO") != "PPO":
            raise NotImplementedError(f"the fused learner runs rsl_rl's ActorCritic + PPO, not {pol.get('class_name')} + {alg.get('class_name')}")
        return SimpleNamespace(cfg=cfg, num_steps_per_env=int(cfg["num_steps_per_env"]), save_interval=int(cfg["save_interval"]),
                               activation=activation_from_rsl_rl(SimpleNamespace(**pol)),
                               init_noise_std=float(pol.get("init_noise_std", 1.0)), alg_cfg=PPOConfig.from_rsl_rl(SimpleNamespace(**alg)))

    def __init__(self, env, train_cfg, log_dir: str | None = None, device="cuda:0"):
        from .policy import pack_actor_critic
        s = self.settings(train_cfg)
        self.env = getattr(env, "unwrapped", env)
        e = self.env
        if getattr(e, "_py_obs", None):
            raise NotImplementedError("Python observation terms (add_observation_term) widen the observation past the slab row the "
                                      "staged step writes: an env with host-side Python terms trains with reward and termination terms only")
        self.staged = bool(getattr(e, "_py_rewards", None) or getattr(e, "_py_terms", None) or getattr(e, "_py_events", None))
        self.dev_names = e.device_log_names if getattr(e, "_dev_terms", None) else []
        dev_step = bool(self.dev_names or getattr(e, "_dev_events", None))     # the rollout steps through wl_step_terms
        sim = e.sim
        if torch.device(device) != torch.device(sim.device):
            raise ValueError(f"device {device} is not the env's device {sim.device}")
        self.critic_obs_dim = sim.critic_obs_dim if getattr(e, "_critic_terms", None) else None
        if self.critic_obs_dim is not None:
            if self.staged:
                raise NotImplementedError("a critic observation group together with host-side Python terms is not implemented")
            if dev_step:
                raise NotImplementedError("a critic observation group together with device terms is not implemented")
            if s.activation != "elu" and sim.policy_width <= 16:
                raise NotImplementedError('a critic observation group with activation="relu" is not implemented for the Drift family '
                                          '(ELU only)')
            if _world_size() > 1:                           # (before anything initialises NCCL)
                raise NotImplementedError("a critic observation group in a data-parallel world (WORLD_SIZE > 1) is not implemented: "
                                          "the exchange buffer is sized by one obs_dim")
        if self.staged and _world_size() > 1:               # (before anything initialises NCCL)
            raise NotImplementedError("data-parallel training of an env with host-side Python terms is not supported: the staged "
                                      "rollout runs on one GPU")
        self.world, self.rank = _data_parallel_world(sim, device)
        self.cfg, self.device, self.log_dir = s.cfg, sim.device, log_dir
        self.num_steps_per_env, self.save_interval, self.activation, self.alg_cfg = s.num_steps_per_env, s.save_interval, s.activation, s.alg_cfg
        D = sim.policy_width                          # (the policy table's width, DESIGN 6q, else the built-in row's)
        if self.activation == "elu" and D > 16:
            raise NotImplementedError(f"the ELU network takes a policy row of at most 16 floats, not {D} (the policy table's width; "
                                      'activation="relu" takes up to 32)')
        act = torch.nn.ELU if self.activation == "elu" else torch.nn.ReLU
        mk = lambda out, nin=D: torch.nn.Sequential(torch.nn.Linear(nin, 64), act(), torch.nn.Linear(64, 64), act(), torch.nn.Linear(64, out))
        std = torch.full((2,), s.init_noise_std)
        self.blob = pack_actor_critic(mk(2), mk(1, self.critic_obs_dim or D), std, D, sim.device, critic_obs_dim=self.critic_obs_dim)
        if self.critic_obs_dim is not None:
            self.it = PPOIteration(sim, self.blob, self.alg_cfg, self.num_steps_per_env, self.activation, episode_stats=True, critic=True)
        elif self.staged:
            self.it = StagedPPOIteration(e, self.blob, self.alg_cfg, self.num_steps_per_env, self.activation)
        else:
            exchange = PPOExchange.symmetric(D, sim.device) if self.world > 1 else None
            self.it = device_terms_iteration(e, self.blob, self.alg_cfg, self.num_steps_per_env, self.activation, exchange) \
                if dev_step else PPOIteration(sim, self.blob, self.alg_cfg, self.num_steps_per_env, self.activation,
                                                    episode_stats=True, exchange=exchange)
        self.alg = self.it.ppo
        self.current_learning_iteration = 0
        self.callback = None
        self.last_log = None

    def learn(self, num_learning_iterations: int, init_at_random_ep_len: bool = False):
        """modified_rsl_rl_runner.py:34-127: iterations current_learning_iteration .. + num_learning_iterations - 1.  The
        episode carries and deques start empty (the runner's locals), the step counter continues from
        ``env.common_step_counter`` and is written back after every iteration; ``model_{it}.pt`` goes to
        ``log_dir/models/`` when ``it % save_interval == 0``."""
        env, it, T = self.env, self.it, self.num_steps_per_env
        if getattr(env, "_needs_reset", False):
            env.reset()
        if init_at_random_ep_len:
            env.episode_length_buf = torch.randint_like(env.episode_length_buf, high=int(env.max_episode_length))
        it.episodes.reset()
        if self.world > 1:
            import torch.distributed as dist
            dist.broadcast(self.blob, src=0)          # every replica starts from rank 0's weights (rsl_rl's learn)
        it.start(env.common_step_counter, capture=True)
        names = sorted(env._log_index.items(), key=lambda kv: kv[1])
        ns = C.sizeof(WlEpisodeStatsState)
        start_iter = self.current_learning_iteration
        for k in range(start_iter, start_iter + num_learning_iterations):
            t0 = time.perf_counter()
            it.run()
            env.sim.flush_log()                       # publish the rollout's last episode-log row into the read-back block
            rb = it.readback.cpu()
            elapsed = time.perf_counter() - t0
            if it.ppo.exchange is not None:
                it.ppo.exchange.check()
            if not self.staged:                       # (the staged step advances the env's counter itself, once per step)
                env.common_step_counter += T
            self.current_learning_iteration = k
            st = WlEpisodeStatsState.from_buffer_copy(bytes(rb[:ns].numpy()))
            summary = rb[ns:ns + 4 * len(PPOIteration.SUMMARY)].view(torch.float32).tolist()
            o_logs = ns + 4 * len(PPOIteration.SUMMARY)
            logs = rb[o_logs:o_logs + 4 * 16 * T].view(torch.float32).view(T, 16).double().mean(0).tolist()
            log = dict(zip(PPOIteration.SUMMARY, summary))
            if st.fill > 0:
                log["Train/mean_reward"] = st.mean_return
                log["Train/mean_episode_length"] = st.mean_length
            log.update({name: logs[col] for name, col in names})
            if self.dev_names:                        # the device terms' entries: T-step means of env.step's extras["log"]
                dev = rb[rb.numel() - 4 * 8 * T:].view(torch.float32).view(T, 8)[:, :len(self.dev_names)].double().mean(0).tolist()
                log.update(zip(self.dev_names, dev))
            if self.staged and it.roll.py_names:      # the Python terms' entries: T-step means of env.step's extras["log"]
                py = rb[rb.numel() - 8 * T * len(it.roll.py_names):].view(torch.float64).view(T, -1).mean(0).tolist()
                log.update(zip(it.roll.py_names, py))
            log["Perf/total_fps"] = T * env.num_envs * self.world / elapsed
            log["Episodes/finished"] = st.finished
            self.last_log = log
            if self.rank != 0:
                continue
            if self.log_dir is not None and k % self.save_interval == 0:
                self.save(os.path.join(self.log_dir, "models", f"model_{k}.pt"))
            if self.callback is not None:
                self.callback(k, log)
        return self.last_log

    def get_inference_policy(self, device=None):
        """rsl_rl's ``get_inference_policy``: ``policy(obs) -> actions``, the actor mean (``policy.InferencePolicy``) over the
        runner's live blob with the runner's activation, so later ``learn`` / ``load`` calls are seen.  The policy runs on
        the env's device: another `device` raises."""
        from .policy import InferencePolicy
        if device is not None:
            norm = lambda x: (x.type, x.index if x.index is not None or x.type != "cuda" else torch.cuda.current_device())
            if norm(torch.device(device)) != norm(torch.device(self.device)):
                raise ValueError(f"device {device} is not the env's device {self.device}: the policy runs where the env's blob is")
        return InferencePolicy(self.blob, self.env.sim.policy_width, self.activation, self.critic_obs_dim)

    def save(self, path: str, infos=None):
        """rsl_rl's checkpoint: {"model_state_dict", "optimizer_state_dict", "iter", "infos"}."""
        from .policy import actor_critic_state_dict
        os.makedirs(os.path.dirname(os.path.abspath(path)), exist_ok=True)
        torch.save({"model_state_dict": actor_critic_state_dict(self.blob, self.env.sim.policy_width, self.critic_obs_dim),
                    "optimizer_state_dict": self.alg.optimizer_state_dict(),
                    "iter": self.current_learning_iteration, "infos": infos}, path)

    def load(self, path: str, load_optimizer: bool = True):
        """Load a checkpoint written by ``save`` or by rsl_rl into the blob (and the Adam state) in place; the next ``learn``
        starts at its ``iter``.  Returns its ``infos``.  A checkpoint whose actor or critic width is not the env's raises
        ``ValueError`` before anything is written -- except with ``load_optimizer=False`` on an env without a critic group,
        where a checkpoint of the asymmetric network loads its actor alone (what ``get_inference_policy`` and playback read)."""
        from .policy import load_actor_critic_state_dict
        d = torch.load(path, map_location=self.device)
        if not isinstance(d, dict) or not {"model_state_dict", "iter"} <= set(d) or (load_optimizer and "optimizer_state_dict" not in d):
            raise ValueError(f"{path}: not an rsl_rl checkpoint (model_state_dict, optimizer_state_dict, iter, infos)")
        D = self.env.sim.policy_width
        try:
            w1 = d["model_state_dict"]["critic.0.weight"]
            # playback of an asymmetric checkpoint on an env without the critic group (play_policy.py loads weights only):
            # the actor is all that plays, so the critic of another width is left out instead of refused
            actor_only = not load_optimizer and self.critic_obs_dim is None and w1.dim() == 2 and w1.shape[1] != D
            blob = load_actor_critic_state_dict(d["model_state_dict"], D, out=self.blob.clone() if actor_only else torch.zeros_like(self.blob),
                                                critic_obs_dim=self.critic_obs_dim, actor_only=actor_only)
        except (KeyError, TypeError, RuntimeError) as e:
            raise ValueError(f"{path}: malformed model_state_dict: {e!r}") from None
        if load_optimizer:
            self.alg.load_optimizer_state_dict(d["optimizer_state_dict"])
        self.blob.copy_(blob)
        self.current_learning_iteration = int(d["iter"])
        return d.get("infos")
