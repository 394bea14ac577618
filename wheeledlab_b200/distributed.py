"""Multi-GPU sharding of the env set (SURVEY 8e) -- one process per GPU, torch.distributed plumbing.

Envs never interact (env_spacing = 0 with inter-env collisions filtered, mushr_drift_env_cfg.py:373), so rank r
owns global env ids [r*N_local, (r+1)*N_local); RNG and domain randomisation are keyed by the GLOBAL id, which makes
the concatenation of the shards bit-identical to one big run.  There is no data-path collective in the step.  The
only exchange is the learner-facing ALL-GATHER of the rollout slab once per PPO iteration (rsl_rl RolloutStorage
consumes [T, N, ...]); the step kernel writes observations / rewards / dones straight into the slab rows, so the
slab IS the send buffer (no staging copy).
"""
from __future__ import annotations

import torch
import torch.distributed as dist


def shard_offset(rank: int, envs_per_rank: int) -> int:
    return rank * envs_per_rank


class RolloutSlab:
    """Per-rank rollout buffer in the layout the learner consumes.  Observations are ONE [T+1,N,D] block: ``obs_in[k]`` (rows
    0..T-1) is the observation the policy saw when it produced ``actions[k]`` -- rsl_rl RolloutStorage.observations[k] --
    and ``obs[k]`` (rows 1..T) is what env.step k returned, so ``obs[k] is obs_in[k+1]`` and ``obs[T-1]`` is the
    bootstrap observation (``obs_in[0]`` must be filled with the rollout's first observation by the caller).
    Other fields: actions [T,N,A] f32,
    rewards [T,N] f32, terminated / truncated [T,N] u8 and -- with ``policy_fields`` -- what alg.act() records per step
    (rsl_rl RolloutStorage: values [T,N], actions_log_prob [T,N], action_mean [T,N,A]; written by wl_act_step).  Fields are
    views of ONE flat byte buffer, so ONE all_gather_into_tensor moves the whole slab.

    ``critic_obs_dim`` (the asymmetric actor-critic, one GPU) adds ``critic_obs_in`` [T+1, N, Dc], the critic rows: row k is
    what ``values[k]`` was computed from, row T the bootstrap row.  It is a tensor of its own, NOT part of ``flat``: the
    asymmetric network is refused in a data-parallel world, so no gather has to carry it; ``critic_obs_in`` is None otherwise.

    ``teacher_actions=True`` (distillation, one GPU) adds ``teacher_actions`` [T, N, A], the teacher's action for the
    observation of step k (rsl_rl RolloutStorage.privileged_actions), likewise a tensor of its own; None otherwise."""

    def __init__(self, T: int, n_local: int, obs_dim: int, act_dim: int, device, policy_fields: bool = False, flat: torch.Tensor | None = None,
                 critic_obs_dim: int | None = None, teacher_actions: bool = False):
        self.T, self.n, self.obs_dim, self.act_dim = T, n_local, obs_dim, act_dim
        self.device = torch.device(device)
        self.teacher_actions = (torch.zeros((T, n_local, act_dim), dtype=torch.float32, device=self.device)
                                if teacher_actions else None)
        self.critic_obs_in = (torch.zeros((T + 1, n_local, critic_obs_dim), dtype=torch.float32, device=self.device)
                              if critic_obs_dim else None)
        # name -> (dtype, trailing shape)
        self._fields = {"obs": (torch.float32, (obs_dim,)), "actions": (torch.float32, (act_dim,)), "rewards": (torch.float32, ()),
                        "terminated": (torch.uint8, ()), "truncated": (torch.uint8, ())}
        if policy_fields:
            self._fields.update({"values": (torch.float32, ()), "log_prob": (torch.float32, ()), "mean": (torch.float32, (act_dim,))})
        f = T * n_local
        self._sizes = {}
        for k, (dt, tail) in self._fields.items():
            n_el = f if k != "obs" else (T + 1) * n_local
            for d in tail:
                n_el *= d
            self._sizes[k] = n_el * (4 if dt == torch.float32 else 1)
        total = sum((v + 255) // 256 * 256 for v in self._sizes.values())
        if flat is not None:                     # caller-provided storage (a slot of a symmetric buffer)
            if flat.numel() != total or flat.dtype != torch.uint8:
                raise ValueError(f"flat must be uint8[{total}]")
            self.flat = flat
        else:
            self.flat = torch.zeros(total, dtype=torch.uint8, device=self.device)
        off = 0
        for k, nbytes in self._sizes.items():
            dt, tail = self._fields[k]
            raw = self.flat[off: off + nbytes]
            if k == "obs":
                self.obs_all = raw.view(torch.float32).view(T + 1, n_local, *tail)
                self.obs_in, self.obs = self.obs_all[:T], self.obs_all[1:]
            else:
                setattr(self, k, (raw.view(torch.float32) if dt == torch.float32 else raw).view(T, n_local, *tail))
            off += (nbytes + 255) // 256 * 256

    @property
    def nbytes(self) -> int:
        return self.flat.numel()

    def step_outputs(self, t: int):
        """Row t as the (obs, rew, terminated, truncated) tuple WheeledSim.step(out=...) writes into."""
        return self.obs[t], self.rewards[t], self.terminated[t], self.truncated[t]

    def all_gather(self, group=None) -> "GatheredRollout":
        """ONE collective: every rank receives every rank's slab (NCCL over NVLink on GPUs, gloo in CPU tests).
        The receive buffer is allocated once and reused: the returned views are overwritten by the next gather (a fresh
        cudaMalloc of world x slab bytes per iteration costs tens of ms)."""
        world = dist.get_world_size(group) if dist.is_initialized() else 1
        if getattr(self, "_recv", None) is None or self._recv.numel() != world * self.flat.numel():
            self._recv = torch.empty(world * self.flat.numel(), dtype=torch.uint8, device=self.device)
        out = self._recv
        if world == 1:
            out.copy_(self.flat)
        else:
            dist.all_gather_into_tensor(out, self.flat, group=group)
        return GatheredRollout(out.view(world, -1), self)


def slab_nbytes(T: int, n_local: int, obs_dim: int, act_dim: int, policy_fields: bool = False) -> int:
    """Size in bytes of a RolloutSlab with this geometry."""
    sizes = [(T + 1) * n_local * obs_dim * 4, T * n_local * act_dim * 4, T * n_local * 4, T * n_local, T * n_local]
    if policy_fields:
        sizes += [T * n_local * 4, T * n_local * 4, T * n_local * act_dim * 4]
    return sum((v + 255) // 256 * 256 for v in sizes)


class SymmetricRolloutSlab:
    """The fused form of the rollout-slab exchange: ONE symmetric (P2P-mapped over NVLink) buffer of world x slab bytes per
    rank (torch.distributed._symmetric_memory).  Rank r's slab is slot r of its own buffer; the step kernel stores every
    output row there AND at the same offset of every peer's buffer (WheeledSim.set_peer_fanout), so after the last step of
    the rollout plus one barrier every rank holds the concatenated rollout -- no all-gather, no staging copy, the transfer
    rides along with the steps.  ``slab`` is the local RolloutSlab, ``gathered()`` the [world, ...] views.  Only
    ``sim.step`` (Drift family, the 8-envs-per-CTA kernel) carries the fan-out, and only the obs, rewards, terminated and
    truncated rows: while a slab is attached, the rollout, act-step, staged and host-transport steps raise WlError.  The
    other fields (actions, policy fields) are the caller's to exchange."""

    def __init__(self, T: int, n_local: int, obs_dim: int, act_dim: int, device, group=None, policy_fields: bool = False):
        import torch.distributed._symmetric_memory as symm
        group = group if group is not None else dist.group.WORLD
        self.world, self.rank = dist.get_world_size(group), dist.get_rank(group)
        nbytes = slab_nbytes(T, n_local, obs_dim, act_dim, policy_fields)
        self.buf = symm.empty(self.world * nbytes, dtype=torch.uint8, device=torch.device(device))
        self.buf.zero_()
        self.handle = symm.rendezvous(self.buf, group.group_name)
        self.slab = RolloutSlab(T, n_local, obs_dim, act_dim, device, policy_fields, flat=self.buf[self.rank * nbytes:(self.rank + 1) * nbytes])
        ptrs = [int(p) for p in self.handle.buffer_ptrs]
        self.peer_deltas = [ptrs[p] - ptrs[self.rank] for p in range(self.world) if p != self.rank]
        mc = int(getattr(self.handle, "multicast_ptr", 0) or 0)    # NVSwitch multicast alias of the buffer (0: not available)
        self.mc_delta = (mc - ptrs[self.rank]) if mc else 0

    def attach(self, sim, multicast: bool = True):
        """Route the step outputs of `sim` to every peer as well."""
        sim.set_peer_fanout(self.peer_deltas)
        sim.set_multicast_fanout(self.mc_delta if multicast else 0)
        return self

    def barrier(self):
        """All ranks' steps issued so far have completed and their peer stores are visible (device-side barrier on the
        current stream; the host is not blocked)."""
        self.handle.barrier()

    def gather_ce(self) -> "GatheredRollout":
        """Pull form of the exchange, on the COPY ENGINES: after a device-side barrier (every rank's slab is complete) each rank
        copies slot p of peer p's buffer into slot p of its own with plain P2P memcpys over NVLink -- no SM is used, so the
        step kernels of the next iteration run undisturbed -- and a second barrier releases the slabs for refilling.  Issued
        on the current stream."""
        nb = self.slab.nbytes
        self.handle.barrier()
        for p in range(self.world):
            if p != self.rank:
                src = self.handle.get_buffer(p, (nb,), torch.uint8, p * nb)
                self.buf[p * nb:(p + 1) * nb].copy_(src, non_blocking=True)
        self.handle.barrier()
        return self.gathered()

    def gathered(self) -> "GatheredRollout":
        return GatheredRollout(self.buf.view(self.world, -1), self.slab)


class GatheredRollout:
    """Views [world, T, N_local, ...] of the gathered bytes; .cat(name) gives the learner's [T, world*N_local, ...]
    with global env id = rank*N_local + local id."""

    def __init__(self, buf: torch.Tensor, proto: RolloutSlab):
        self.buf, self.p = buf, proto

    def field(self, name: str) -> torch.Tensor:
        p = self.p
        if name == "obs_in":
            off = 0
            for k, nbytes in p._sizes.items():
                if k == "obs":
                    break
                off += (nbytes + 255) // 256 * 256
            raw = self.buf[:, off: off + p._sizes["obs"]]
            return raw.view(torch.float32).view(self.buf.shape[0], p.T + 1, p.n, p.obs_dim)[:, :p.T]
        off = 0
        for k, nbytes in p._sizes.items():
            if k == name:
                raw = self.buf[:, off: off + nbytes]
                break
            off += (nbytes + 255) // 256 * 256
        else:
            raise KeyError(name)
        dt, tail = p._fields[name]
        if name == "obs":                          # rows 1..T of the [T+1] block (see RolloutSlab); "obs_in" = rows 0..T-1
            return raw.view(torch.float32).view(self.buf.shape[0], p.T + 1, p.n, *tail)[:, 1:]
        return (raw.view(torch.float32) if dt == torch.float32 else raw).view(self.buf.shape[0], p.T, p.n, *tail)

    def cat(self, name: str) -> torch.Tensor:
        f = self.field(name)                       # [W, T, N, ...] -> [T, W*N, ...]
        return f.transpose(0, 1).reshape(f.shape[1], f.shape[0] * f.shape[2], *f.shape[3:])
