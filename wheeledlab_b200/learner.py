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

from ._lib import WlEpisodeStatsState, WlError, WlPpoBatch, WlPpoParams, check, lib


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

    def optimizer_state_dict(self) -> dict:
        """What ``torch.optim.Adam(actor_critic.parameters()).state_dict()`` holds in rsl_rl's checkpoints
        (``optimizer_state_dict``): params 0..12 in ActorCritic order (actor.0/2/4 weight|bias, critic.0/2/4 weight|bias,
        std), ``state[i] = {step, exp_avg, exp_avg_sq}`` with the moments transposed out of the blob layout as
        ``policy.actor_critic_state_dict`` does for the weights (empty before the first update), and one param group with
        the current learning rate.  Reads the device state (one sync)."""
        from .policy import actor_critic_state_dict
        lr, step = (float(x) for x in self.state[:2].tolist())
        m, v = actor_critic_state_dict(self.m, self.obs_dim), actor_critic_state_dict(self.v, self.obs_dim)
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
        names = list(actor_critic_state_dict(self.m, self.obs_dim))
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
                    load_actor_critic_state_dict({k: st[i][key] for i, k in enumerate(names)}, self.obs_dim, out=out)
            except (KeyError, TypeError, RuntimeError) as e:
                raise ValueError(f"malformed optimizer state: {e!r}") from None
            if len(steps) != 1:
                raise ValueError(f"the 13 parameters have different Adam step counts {sorted(steps)}")
            step = steps.pop()
        self.m.copy_(m)
        self.v.copy_(v)
        self.state[1] = step
        self.state[0] = self.cfg.learning_rate


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
    it), so that one copy reads an iteration back."""

    SUMMARY = ("Loss/value_function", "Loss/surrogate", "Loss/entropy", "Loss/learning_rate", "Policy/mean_noise_std")

    def __init__(self, sim, blob: torch.Tensor, cfg: PPOConfig | None = None, T: int = 128, activation: str = "elu",
                 episode_stats: bool = False):
        from .policy import FusedPolicyRollout
        self.sim, self.blob, self.T = sim, blob, T
        self.roll = FusedPolicyRollout(sim, blob, T, activation=activation)
        self.ppo = FusedPPO(blob, sim.obs_dim, cfg, activation)
        self.perm = torch.empty(T * sim.num_envs, dtype=torch.int64, device=sim.device)
        self.graph = None
        self.stats = None
        self.episodes = self.readback = self.summary = None
        if episode_stats:
            ns = C.sizeof(WlEpisodeStatsState)
            self.readback = torch.zeros(ns + 4 * len(self.SUMMARY) + 4 * 16 * T, dtype=torch.uint8, device=sim.device)
            self.episodes = EpisodeStatistics(sim.num_envs, T, sim.device, state=self.readback[:ns])
            self.summary = self.readback[ns:ns + 4 * len(self.SUMMARY)].view(torch.float32)
            self.roll.logs = self.readback[ns + 4 * len(self.SUMMARY):].view(torch.float32).view(T, 16)

    def _bootstrap(self) -> torch.Tensor:
        from .policy import critic_value
        return critic_value(self.blob, self.sim.obs_dim, self.roll.obs0, self.ppo.activation)

    def _learn(self):
        slab, cfg = self.roll.slab, self.ppo.cfg
        if self.episodes is not None:
            self.episodes.update(slab.rewards, slab.terminated, slab.truncated)
        last_values = self._bootstrap()
        ret, adv = compute_returns(slab.rewards, slab.values, last_values, slab.terminated | slab.truncated, cfg.gamma, cfg.lam,
                                   time_outs=slab.truncated)
        stats = self.ppo.update(slab, ret, adv, self.perm)
        if self.summary is not None:
            from .policy import blob_layout
            o_std = blob_layout(self.sim.obs_dim)[0][12]
            self.summary.copy_(torch.stack([stats["value_function"], stats["surrogate"], stats["entropy"], stats["learning_rate"],
                                            self.blob[o_std:o_std + 2].mean()]))
        return stats

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


class FusedOnPolicyRunner:
    """rsl_rl's ``OnPolicyRunner`` as the reference drives it (``modified_rsl_rl_runner.py``, ``train_rl.py:95-116``), over
    ``PPOIteration``: ``FusedOnPolicyRunner(env, agent_cfg.to_dict(), log_dir, device)``, ``learn(n)``, ``save`` / ``load``
    in rsl_rl's checkpoint format.  ``env`` is a ``wheeledlab_b200.env.ManagerBasedRLEnv`` (or a wrapper whose ``unwrapped``
    is one) without host-side Python terms.  Each iteration is ONE CUDA graph -- rollout, ``wl_episode_stats``, bootstrap
    value, GAE, PPO update -- plus the flush of the last episode-log row, and ONE read-back of what is logged.

    The agent cfg dict is read for ``num_steps_per_env``, ``save_interval``, ``policy`` (``activation_from_rsl_rl``,
    ``init_noise_std``) and ``algorithm`` (``PPOConfig.from_rsl_rl``).  The weights start as the reference's do: torch
    ``nn.Linear`` defaults from torch's global generator, std = ``init_noise_std``.  No writer: ``callback(it, scalars)``,
    if set, receives each iteration's scalars (also kept in ``self.last_log``)."""

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
        if getattr(e, "_py_rewards", None) or getattr(e, "_py_terms", None) or getattr(e, "_py_obs", None):
            raise NotImplementedError("the fused rollout runs the kernels' MDP terms only: this env has host-side Python terms")
        sim = e.sim
        if torch.device(device) != torch.device(sim.device):
            raise ValueError(f"device {device} is not the env's device {sim.device}")
        self.cfg, self.device, self.log_dir = s.cfg, sim.device, log_dir
        self.num_steps_per_env, self.save_interval, self.activation, self.alg_cfg = s.num_steps_per_env, s.save_interval, s.activation, s.alg_cfg
        D = sim.obs_dim
        act = torch.nn.ELU if self.activation == "elu" else torch.nn.ReLU
        mk = lambda out: torch.nn.Sequential(torch.nn.Linear(D, 64), act(), torch.nn.Linear(64, 64), act(), torch.nn.Linear(64, out))
        std = torch.full((2,), s.init_noise_std)
        self.blob = pack_actor_critic(mk(2), mk(1), std, D, sim.device)
        self.it = PPOIteration(sim, self.blob, self.alg_cfg, self.num_steps_per_env, self.activation, episode_stats=True)
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
            env.common_step_counter += T
            self.current_learning_iteration = k
            st = WlEpisodeStatsState.from_buffer_copy(bytes(rb[:ns].numpy()))
            summary = rb[ns:ns + 4 * len(PPOIteration.SUMMARY)].view(torch.float32).tolist()
            logs = rb[ns + 4 * len(PPOIteration.SUMMARY):].view(torch.float32).view(T, 16).double().mean(0).tolist()
            log = dict(zip(PPOIteration.SUMMARY, summary))
            if st.fill > 0:
                log["Train/mean_reward"] = st.mean_return
                log["Train/mean_episode_length"] = st.mean_length
            log.update({name: logs[col] for name, col in names})
            log["Perf/total_fps"] = T * env.num_envs / elapsed
            log["Episodes/finished"] = st.finished
            self.last_log = log
            if self.log_dir is not None and k % self.save_interval == 0:
                self.save(os.path.join(self.log_dir, "models", f"model_{k}.pt"))
            if self.callback is not None:
                self.callback(k, log)
        return self.last_log

    def save(self, path: str, infos=None):
        """rsl_rl's checkpoint: {"model_state_dict", "optimizer_state_dict", "iter", "infos"}."""
        from .policy import actor_critic_state_dict
        os.makedirs(os.path.dirname(os.path.abspath(path)), exist_ok=True)
        torch.save({"model_state_dict": actor_critic_state_dict(self.blob, self.env.sim.obs_dim),
                    "optimizer_state_dict": self.alg.optimizer_state_dict(),
                    "iter": self.current_learning_iteration, "infos": infos}, path)

    def load(self, path: str, load_optimizer: bool = True):
        """Load a checkpoint written by ``save`` or by rsl_rl into the blob (and the Adam state) in place; the next ``learn``
        starts at its ``iter``.  Returns its ``infos``."""
        from .policy import load_actor_critic_state_dict
        d = torch.load(path, map_location=self.device)
        if not isinstance(d, dict) or not {"model_state_dict", "iter"} <= set(d) or (load_optimizer and "optimizer_state_dict" not in d):
            raise ValueError(f"{path}: not an rsl_rl checkpoint (model_state_dict, optimizer_state_dict, iter, infos)")
        D = self.env.sim.obs_dim
        try:
            blob = load_actor_critic_state_dict(d["model_state_dict"], D, out=torch.zeros_like(self.blob))
        except (KeyError, TypeError, RuntimeError) as e:
            raise ValueError(f"{path}: malformed model_state_dict: {e!r}") from None
        if load_optimizer:
            self.alg.load_optimizer_state_dict(d["optimizer_state_dict"])
        self.blob.copy_(blob)
        self.current_learning_iteration = int(d["iter"])
        return d.get("infos")
