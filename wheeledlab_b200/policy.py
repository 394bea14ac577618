"""The policy side of the rollout loop, fused in front of the env step (SURVEY 8f-1).

``alg.act(obs)`` (modified_rsl_rl_runner.py:72) evaluates rsl_rl's ActorCritic [UPSTREAM-RECALL]: two 64x64 ELU MLPs
(drifting/config/agents/mushr/rsl_rl_ppo_cfg.py:12-17), a Gaussian head with a learned per-action std, and returns the
sampled action while the storage keeps value / mean / std / log-prob.  ``wl_act_step`` does all of that AND the env step in
one launch; this module packs torch ``nn.Linear`` weights into the kernel's blob layout and provides the graph-captured
rollout built on it.
"""
from __future__ import annotations

import ctypes as C
from types import SimpleNamespace

import torch

from ._lib import WL_ACTIVATION, WlPolicyOut, check, lib
from .distributed import RolloutSlab
from .sim import WheeledSim, _stream_ptr

HIDDEN = 64


def blob_layout(obs_dim: int, critic_obs_dim: int | None = None):
    """Offsets and float count of the blob; ``critic_obs_dim`` (None: the critic reads the policy row) sizes the critic's
    first layer for the asymmetric network (wl_policy_blob_floats_asym)."""
    off = (C.c_int32 * 13)()
    if critic_obs_dim is None:
        total = lib.wl_policy_blob_floats(obs_dim, off)
    else:
        total = lib.wl_policy_blob_floats_asym(obs_dim, critic_obs_dim, off)
    return list(off), total


def _linears(net):
    ls = [m for m in net.modules() if isinstance(m, torch.nn.Linear)]
    if len(ls) != 3 or ls[0].out_features != HIDDEN or ls[1].in_features != HIDDEN or ls[1].out_features != HIDDEN:
        raise NotImplementedError("wl_act_step implements the reference's [64, 64] ELU actor / critic only")
    return ls


def pack_actor_critic(actor, critic, std: torch.Tensor, obs_dim: int, device, out: torch.Tensor | None = None,
                      critic_obs_dim: int | None = None) -> torch.Tensor:
    """actor / critic: torch modules holding three nn.Linear (obs->64->64->2 / ->1, ELU in between); std: [2].
    Returns (or refills, when `out` is given -- e.g. after an optimiser step) the fp32 device blob wl_act_step reads.
    ``critic_obs_dim``: the critic's input width when it reads a row of its own (wl_policy_act_asym's blob)."""
    off, total = blob_layout(obs_dim, critic_obs_dim)
    blob = out if out is not None else torch.zeros(total, dtype=torch.float32, device=device)
    with torch.no_grad():
        for net_i, (net, nout) in enumerate(((actor, 2), (critic, 1))):
            ls = _linears(net)
            nin = obs_dim if net_i == 0 or critic_obs_dim is None else critic_obs_dim
            if ls[0].in_features != nin or ls[2].out_features != nout:
                raise ValueError("network shape does not match the task")
            for k, lin in enumerate(ls):
                wt = lin.weight.detach().to(device=device, dtype=torch.float32).t().contiguous().reshape(-1)   # input-major
                o = off[net_i * 6 + 2 * k]
                blob[o:o + wt.numel()].copy_(wt)
                o = off[net_i * 6 + 2 * k + 1]
                blob[o:o + lin.bias.numel()].copy_(lin.bias.detach().to(device=device, dtype=torch.float32))
        blob[off[12]:off[12] + 2].copy_(std.detach().to(device=device, dtype=torch.float32))
    return blob


def _blob_layers(blob: torch.Tensor, obs_dim: int, critic_obs_dim: int | None = None):
    """Zero-copy views of the blob: per net, three (W [in, out] input-major, b [out]) pairs; plus std [2]."""
    off, _ = blob_layout(obs_dim, critic_obs_dim)
    nets = []
    for net_i, nout in enumerate((2, 1)):
        o = off[net_i * 6:net_i * 6 + 6]
        nin = obs_dim if net_i == 0 or critic_obs_dim is None else critic_obs_dim
        nets.append([(blob[o[0]:o[0] + nin * HIDDEN].view(nin, HIDDEN), blob[o[1]:o[1] + HIDDEN]),
                     (blob[o[2]:o[2] + HIDDEN * HIDDEN].view(HIDDEN, HIDDEN), blob[o[3]:o[3] + HIDDEN]),
                     (blob[o[4]:o[4] + HIDDEN * nout].view(HIDDEN, nout), blob[o[5]:o[5] + nout])])
    return nets[0], nets[1], blob[off[12]:off[12] + 2]


def actor_critic_state_dict(blob: torch.Tensor, obs_dim: int, critic_obs_dim: int | None = None) -> dict:
    """The blob as an rsl_rl ActorCritic state dict (actor.0/2/4.weight|bias, critic.0/2/4.weight|bias, std) [UPSTREAM-RECALL]:
    the ``model_state_dict`` of the checkpoints rsl_rl's runner saves and ``play_policy.py`` loads.  Tensors are copies.
    With ``critic_obs_dim`` ``critic.0.weight`` is [64, critic_obs_dim], as ActorCritic(num_actor_obs, num_critic_obs, ...) has it."""
    actor, critic, std = _blob_layers(blob, obs_dim, critic_obs_dim)
    sd = {}
    for name, layers in (("actor", actor), ("critic", critic)):
        for k, (w, b) in enumerate(layers):
            sd[f"{name}.{2 * k}.weight"] = w.t().contiguous()
            sd[f"{name}.{2 * k}.bias"] = b.clone()
    sd["std"] = std.clone()
    return sd


def load_actor_critic_state_dict(sd: dict, obs_dim: int, out: torch.Tensor | None = None, device=None,
                                 critic_obs_dim: int | None = None, actor_only: bool = False) -> torch.Tensor:
    """Inverse of actor_critic_state_dict: fills `out` (or a new zeroed blob) from an rsl_rl ActorCritic state dict.  Every
    shape is checked before anything is written: a checkpoint whose actor or critic width does not match leaves `out` as it was.
    ``actor_only``: the actor blocks and std alone, the critic's neither checked nor written -- what playback needs of a
    checkpoint whose critic read a row of its own (the actor blocks sit at the same offsets in both layouts)."""
    if out is None:
        out = torch.zeros(blob_layout(obs_dim, critic_obs_dim)[1], dtype=torch.float32, device=device or sd["std"].device)
    actor, critic, std = _blob_layers(out, obs_dim, critic_obs_dim)
    nets = (("actor", actor),) if actor_only else (("actor", actor), ("critic", critic))
    for name, layers in nets:
        for k, (w, b) in enumerate(layers):
            wt, bt = sd[f"{name}.{2 * k}.weight"], sd[f"{name}.{2 * k}.bias"]
            if tuple(wt.shape) != (w.shape[1], w.shape[0]) or tuple(bt.shape) != tuple(b.shape):
                width = f"obs_dim {obs_dim}" + ("" if critic_obs_dim is None else f" and critic width {critic_obs_dim}")
                raise ValueError(f"{name}.{2 * k}: shape {tuple(wt.shape)} does not match the [64, 64] ELU network of {width}")
    with torch.no_grad():
        for name, layers in nets:
            for k, (w, b) in enumerate(layers):
                wt, bt = sd[f"{name}.{2 * k}.weight"], sd[f"{name}.{2 * k}.bias"]
                w.copy_(wt.t())
                b.copy_(bt)
        std.copy_(sd["std"])
    return out


ACTIVATIONS = {"elu": torch.nn.functional.elu, "relu": torch.nn.functional.relu}


def check_activation(activation: str) -> str:
    if activation not in ACTIVATIONS:
        raise ValueError(f"activation must be 'elu' (the Drift family's network) or 'relu' (Elevation / Visual), not {activation!r}")
    return activation


def critic_value(blob: torch.Tensor, obs_dim: int, obs: torch.Tensor, activation: str = "elu",
                 critic_obs_dim: int | None = None) -> torch.Tensor:
    """V(obs) [N] in torch from zero-copy views of the blob (the bootstrap value of compute_returns): a CUDA graph that
    captures it reads the weights the last update left in the blob.  With ``critic_obs_dim`` `obs` is the critic row."""
    act = ACTIVATIONS[check_activation(activation)]
    _, critic, _ = _blob_layers(blob, obs_dim, critic_obs_dim)
    x = obs
    for k, (w, b) in enumerate(critic):
        x = torch.addmm(b, x, w)
        if k < 2:
            x = act(x)
    return x.squeeze(-1)


def _device_tensor(name: str, t, device, shape=None, ndim=None) -> None:
    if not isinstance(t, torch.Tensor):
        raise ValueError(f"{name} must be a torch.Tensor")
    if t.device.type != "cuda" or (device is not None and t.device != device):
        raise ValueError(f"{name} must be on {device or 'a CUDA device'}, not {t.device}")
    if t.dtype != torch.float32:
        raise ValueError(f"{name} must be float32, not {t.dtype}")
    if ndim is not None and t.dim() != ndim:
        raise ValueError(f"{name} must have {ndim} dimension(s), not shape {tuple(t.shape)}")
    if shape is not None and tuple(t.shape) != tuple(shape):
        raise ValueError(f"{name} must have shape {tuple(shape)}, not {tuple(t.shape)}")
    if not t.is_contiguous():
        raise ValueError(f"{name} must be contiguous")


def actor_mean(blob: torch.Tensor, obs_dim: int, obs: torch.Tensor, activation: str = "elu", out: torch.Tensor | None = None,
               critic_obs_dim: int | None = None) -> torch.Tensor:
    """The actor mean [N, 2] of `obs` [N, obs_dim] under the network in `blob` -- rsl_rl ``ActorCritic.act_inference``, the
    deterministic action a trained policy is played with.  One launch (wl_actor_mean) on the current stream of obs's
    device; into `out` [N, 2] when given (capturable), else into a new tensor.  "elu": the Drift family's network
    (obs_dim <= 16), bit for bit the mean wl_act_step stores; "relu": Elevation / Visual (obs_dim <= 4096), bit for bit
    wl_policy_act's mean.  ``critic_obs_dim``: the blob is the asymmetric network's (blob_layout(obs_dim, critic_obs_dim));
    the actor blocks sit at the same offsets, so it plays unchanged."""
    check_activation(activation)
    _device_tensor("obs", obs, None, ndim=2)
    dev = obs.device
    if obs.shape[1] != obs_dim:
        raise ValueError(f"obs must have shape [N, {obs_dim}], not {tuple(obs.shape)}")
    if obs.shape[0] < 1:
        raise ValueError("obs must have at least one row")
    _device_tensor("blob", blob, dev, shape=(blob_layout(obs_dim, critic_obs_dim)[1],))
    if out is None:
        out = torch.empty((obs.shape[0], 2), dtype=torch.float32, device=dev)
    else:
        _device_tensor("out", out, dev, shape=(obs.shape[0], 2))
    check(lib.wl_actor_mean(C.c_void_p(obs.data_ptr()), obs.shape[0], obs_dim, C.c_void_p(blob.data_ptr()), WL_ACTIVATION[activation],
                            C.c_void_p(out.data_ptr()), _stream_ptr(dev)), "wl_actor_mean")
    return out


class InferencePolicy:
    """rsl_rl's ``runner.get_inference_policy()``: ``policy(obs) -> actions [N, 2]``, the actor mean (actor_mean), a new
    tensor per call (play_policy.py appends the actions without cloning) unless `out` is given.  The blob is read at call
    time, so later updates and loads into it are seen.  Works under ``torch.inference_mode()``."""

    def __init__(self, blob: torch.Tensor, obs_dim: int, activation: str = "elu", critic_obs_dim: int | None = None):
        self.blob, self.obs_dim, self.activation, self.critic_obs_dim = blob, obs_dim, check_activation(activation), critic_obs_dim

    def __call__(self, obs: torch.Tensor, out: torch.Tensor | None = None) -> torch.Tensor:
        return actor_mean(self.blob, self.obs_dim, obs, self.activation, out, self.critic_obs_dim)


class PolicyBuffers:
    """[T, N] storage of what alg.act() records per step (rsl_rl RolloutStorage fields)."""

    def __init__(self, T: int, N: int, device):
        self.mean = torch.zeros((T, N, 2), dtype=torch.float32, device=device)
        self.log_prob = torch.zeros((T, N), dtype=torch.float32, device=device)
        self.values = torch.zeros((T, N), dtype=torch.float32, device=device)


def act_step(sim: WheeledSim, obs_in: torch.Tensor, blob: torch.Tensor, actions: torch.Tensor, mean: torch.Tensor,
             log_prob: torch.Tensor, value: torch.Tensor, out, log: torch.Tensor | None, step_counter: int):
    """One launch: value/mean/sample/log-prob of `obs_in` under `blob`, then env.step(sampled action) into `out`."""
    obs, rew, term, trunc = out
    po = WlPolicyOut(actions.data_ptr(), mean.data_ptr(), log_prob.data_ptr(), value.data_ptr())
    check(lib.wl_act_step(sim._h, C.c_void_p(obs_in.data_ptr()), C.c_void_p(blob.data_ptr()), po, C.c_void_p(obs.data_ptr()),
                          C.c_void_p(rew.data_ptr()), C.c_void_p(term.data_ptr()), C.c_void_p(trunc.data_ptr()),
                          C.c_void_p(log.data_ptr()) if log is not None else None, step_counter, _stream_ptr(sim.device)),
          "wl_act_step")


def act_infer_step(sim: WheeledSim, obs_in: torch.Tensor, blob: torch.Tensor, actions: torch.Tensor, out, log: torch.Tensor | None,
                   step_counter: int):
    """One launch (wl_act_infer_step): the actor mean of `obs_in` under the ELU network in `blob` into `actions`, then
    env.step(actions) into `out`."""
    obs, rew, term, trunc = out
    check(lib.wl_act_infer_step(sim._h, C.c_void_p(obs_in.data_ptr()), C.c_void_p(blob.data_ptr()), C.c_void_p(actions.data_ptr()),
                                C.c_void_p(obs.data_ptr()), C.c_void_p(rew.data_ptr()), C.c_void_p(term.data_ptr()),
                                C.c_void_p(trunc.data_ptr()), C.c_void_p(log.data_ptr()) if log is not None else None, step_counter,
                                _stream_ptr(sim.device)), "wl_act_infer_step")


def policy_act(sim: WheeledSim, obs_in: torch.Tensor, blob: torch.Tensor, actions: torch.Tensor, mean: torch.Tensor,
               log_prob: torch.Tensor, value: torch.Tensor, step_counter: int, activation: str = "relu"):
    """One launch: value / mean / sample / log-prob of `obs_in` [N, obs_dim] under the network in `blob`.  "relu"
    (wl_policy_act): Elevation / Visual, any obs_dim up to 4096; "elu" (wl_policy_act_elu): the Drift family's network
    (obs_dim <= 16), bit for bit what wl_act_step stores.  The env is not stepped: follow with a step on the same
    step_counter (sim.step, or the staged step)."""
    fn = lib.wl_policy_act if check_activation(activation) == "relu" else lib.wl_policy_act_elu
    po = WlPolicyOut(actions.data_ptr(), mean.data_ptr(), log_prob.data_ptr(), value.data_ptr())
    check(fn(sim._h, C.c_void_p(obs_in.data_ptr()), C.c_void_p(blob.data_ptr()), po, step_counter, _stream_ptr(sim.device)),
          fn.__name__)


def policy_act_asym(sim: WheeledSim, obs_in: torch.Tensor, critic_obs_in: torch.Tensor, blob: torch.Tensor, actions: torch.Tensor,
                    mean: torch.Tensor, log_prob: torch.Tensor, value: torch.Tensor, step_counter: int):
    """policy_act(..., "elu") for the asymmetric network (wl_policy_act_asym): the critic reads `critic_obs_in` [N, Dc] and the
    blob is laid out by blob_layout(obs_dim, Dc); actions / mean / log-prob are wl_policy_act_elu's bit for bit."""
    n = sim.num_envs
    if critic_obs_in.dim() != 2 or not 1 <= critic_obs_in.shape[1] <= 32:
        raise ValueError(f"critic_obs_in must have shape [N, Dc] with Dc in 1..32, not {tuple(critic_obs_in.shape)}")
    _device_tensor("obs_in", obs_in, sim.device, shape=(n, sim.policy_width))
    _device_tensor("critic_obs_in", critic_obs_in, sim.device, shape=(n, critic_obs_in.shape[1]))
    _device_tensor("blob", blob, sim.device, shape=(blob_layout(sim.policy_width, critic_obs_in.shape[1])[1],))
    for name, t, shape in (("actions", actions, (n, 2)), ("mean", mean, (n, 2)), ("log_prob", log_prob, (n,)), ("value", value, (n,))):
        _device_tensor(name, t, sim.device, shape=shape)
    po = WlPolicyOut(actions.data_ptr(), mean.data_ptr(), log_prob.data_ptr(), value.data_ptr())
    check(lib.wl_policy_act_asym(sim._h, C.c_void_p(obs_in.data_ptr()), C.c_void_p(critic_obs_in.data_ptr()), critic_obs_in.shape[-1],
                                 C.c_void_p(blob.data_ptr()), po, step_counter, _stream_ptr(sim.device)), "wl_policy_act_asym")


def policy_act_wide_asym(sim: WheeledSim, obs_in: torch.Tensor, critic_obs_in: torch.Tensor, blob: torch.Tensor, actions: torch.Tensor,
                         mean: torch.Tensor, log_prob: torch.Tensor, value: torch.Tensor, step_counter: int):
    """policy_act(..., "relu") for the asymmetric network (wl_policy_act_wide_asym, DESIGN 6s): the critic reads
    `critic_obs_in` [N, Dc] (Dc <= 4096, e.g. an Elevation row critic's) and the blob is laid out by blob_layout(obs_dim, Dc);
    actions / mean / log-prob are wl_policy_act's bit for bit."""
    n = sim.num_envs
    if critic_obs_in.dim() != 2 or not 1 <= critic_obs_in.shape[1] <= 4096:
        raise ValueError(f"critic_obs_in must have shape [N, Dc] with Dc in 1..4096, not {tuple(critic_obs_in.shape)}")
    _device_tensor("obs_in", obs_in, sim.device, shape=(n, sim.policy_width))
    _device_tensor("critic_obs_in", critic_obs_in, sim.device, shape=(n, critic_obs_in.shape[1]))
    _device_tensor("blob", blob, sim.device, shape=(blob_layout(sim.policy_width, critic_obs_in.shape[1])[1],))
    for name, t, shape in (("actions", actions, (n, 2)), ("mean", mean, (n, 2)), ("log_prob", log_prob, (n,)), ("value", value, (n,))):
        _device_tensor(name, t, sim.device, shape=shape)
    po = WlPolicyOut(actions.data_ptr(), mean.data_ptr(), log_prob.data_ptr(), value.data_ptr())
    check(lib.wl_policy_act_wide_asym(sim._h, C.c_void_p(obs_in.data_ptr()), C.c_void_p(critic_obs_in.data_ptr()),
                                      critic_obs_in.shape[-1], C.c_void_p(blob.data_ptr()), po, step_counter, _stream_ptr(sim.device)),
          "wl_policy_act_wide_asym")


class FusedPolicyRollout:
    """T policy-and-step launches captured as ONE CUDA graph: the reference's whole collection loop
    (modified_rsl_rl_runner.py:70-109).  activation "elu" (the Drift family): T x wl_act_step, the policy fused into the
    step; "relu" (Elevation, Visual): T x (wl_policy_act, then wl_step).  The blob is read at replay time, so refilling it
    in place (pack_actor_critic(..., out=blob)) after each PPO update needs no re-capture.

    ``deterministic=True`` plays the policy instead (play_policy.py's loop): the action is the actor mean, with no critic and
    no noise -- T x wl_act_infer_step for "elu", T x (wl_actor_mean, then wl_step) for "relu" -- and the slab has no
    policy fields.  ``slab.obs[k]`` / ``slab.actions[k]`` are what play_policy.py appends at step k, so
    ``recording.save_slab(playback_dir, play_name, roll.slab)`` writes its rollouts file.

    ``device_terms=True`` rolls out an env whose handle has device terms (``wl_set_device_terms``): T x (``policy_act``,
    then ``wl_step_terms``) on the same device counters, still one graph; ``term_logs[k]`` [T, 8] receives step k's
    device-term ``Episode_*`` entries.  A graph must be captured after the handle's terms are set.

    ``critic=True`` rolls out the asymmetric network on a handle that has a critic table (``sim.set_critic_terms``): T x
    (``policy_act_asym``, ``wl_step``, ``wl_critic_observe`` into row k + 1) on device counters, one graph.
    ``slab.critic_obs_in`` [T + 1, N, Dc] holds the critic rows: row k is what ``values[k]`` was computed from, row T the
    bootstrap row.  The blob is laid out by ``blob_layout(obs_dim, Dc)``.  Not with device terms.  "elu" for the Drift
    family; "relu" for an Elevation handle with a row critic (``sim.set_row_critic``, DESIGN 6s), with or without row
    terms: T x (``policy_act_wide_asym``, ``wl_step``, ``wl_critic_observe``).

    On a handle with a policy observation table (``sim.set_policy_terms``, DESIGN 6q) every step is the policy kernel of the
    network on ``slab.obs_in[k]`` (``wl_policy_act_elu`` / ``wl_policy_act`` / ``wl_policy_act_asym``, or ``wl_actor_mean``
    when deterministic), the step writing its built-in row to a scratch buffer, then ``wl_policy_observe`` into
    ``slab.obs[k]`` = ``obs_in[k + 1]`` (and ``wl_critic_observe`` with a critic), still one graph; the slab and the blob
    are sized by the table's width."""

    def __init__(self, sim: WheeledSim, blob: torch.Tensor, T: int = 128, slab: RolloutSlab | None = None, activation: str = "elu",
                 deterministic: bool = False, device_terms: bool = False, critic: bool = False):
        self.sim, self.blob, self.T, self.activation = sim, blob, T, check_activation(activation)
        self.deterministic = bool(deterministic)
        self.device_terms = bool(device_terms)
        self.critic = bool(critic)
        if self.critic:
            if self.deterministic:
                raise ValueError("critic: the training rollout only (playback reads the actor alone)")
            if self.device_terms:
                raise NotImplementedError("a critic observation group together with device terms is not implemented")
            if activation != "elu" and sim.policy_width <= 16:
                raise NotImplementedError('a critic observation group with activation="relu" is not implemented for the Drift '
                                          'family (ELU only)')
            if sim.critic_obs_dim < 1:
                raise ValueError("critic=True needs a critic table on the handle (sim.set_critic_terms)")
            if (sim.num_envs * sim.obs_dim) % 2:
                raise ValueError("wl_step writes each slab observation row pair-wise: num_envs * obs_dim must be even")
        if self.device_terms and self.deterministic:
            raise ValueError("device_terms: the training rollout only")
        if self.device_terms and (sim.num_envs * sim.obs_dim) % 2:
            raise ValueError("the slab's observation rows are written pair-wise: num_envs * obs_dim must be even")
        self.term_logs = torch.zeros((T, 8), dtype=torch.float32, device=sim.device) if self.device_terms else None
        if activation == "relu" and (sim.num_envs * sim.obs_dim) % 2:
            raise ValueError("wl_step writes each slab observation row pair-wise: num_envs * obs_dim must be even")
        self.table = sim.policy_obs_dim > 0
        # row terms (DESIGN 6r): the fused act step writes the built-in row, so the policy kernel and wl_step are separate
        self.rows = sim.row_terms > 0
        D = sim.policy_width
        self.slab = slab or RolloutSlab(T, sim.num_envs, D, 2, sim.device, policy_fields=not self.deterministic,
                                        critic_obs_dim=sim.critic_obs_dim if self.critic else None)
        # with a table the step's built-in row is scratch: the policy reads wl_policy_observe's row
        self._scratch = torch.empty((sim.num_envs, sim.obs_dim), dtype=torch.float32, device=sim.device) if self.table else None
        # values / log-prob / mean go straight into the slab (= the all-gather send buffer) when it has those fields
        if self.deterministic:
            self.pol = None
        else:
            self.pol = (SimpleNamespace(values=self.slab.values, log_prob=self.slab.log_prob, mean=self.slab.mean)
                        if hasattr(self.slab, "values") else PolicyBuffers(T, sim.num_envs, sim.device))
        self.logs = torch.zeros((T, 16), dtype=torch.float32, device=sim.device)
        # slab.obs_in[k] = the observation actions[k] / log_prob[k] / values[k] / mean[k] were computed from (rsl_rl
        # RolloutStorage.observations[k]); slab.obs[k] = obs_in[k+1] = what step k returned
        self.obs0 = torch.empty((sim.num_envs, D), dtype=torch.float32, device=sim.device)    # carried to the next replay
        if self.critic:
            if self.slab.critic_obs_in is None or tuple(self.slab.critic_obs_in.shape) != (T + 1, sim.num_envs, sim.critic_obs_dim):
                raise ValueError(f"critic=True needs a slab built with critic_obs_dim={sim.critic_obs_dim}")
            self.cobs0 = torch.empty((sim.num_envs, sim.critic_obs_dim), dtype=torch.float32, device=sim.device)
        self.graph = None
        self._base = 0
        self._stream = torch.cuda.Stream(device=sim.device)

    def _step_outputs(self, k: int):
        """What the step writes at k: the slab's row k, or with a table the scratch row (the table's row follows it)."""
        if not self.table:
            return self.slab.step_outputs(k)
        return (self._scratch,) + self.slab.step_outputs(k)[1:]

    def _table_step(self, k: int, t: int):
        """Step k on a handle with a policy table: the policy kernel, the step into scratch, the table's row into obs_in[k+1]."""
        slab, sim, D = self.slab, self.sim, self.sim.policy_width
        if self.deterministic:
            actor_mean(self.blob, D, slab.obs_in[k], self.activation, out=slab.actions[k])
        elif self.critic:
            act = policy_act_wide_asym if self.activation == "relu" else policy_act_asym
            act(sim, slab.obs_in[k], slab.critic_obs_in[k], self.blob, slab.actions[k], self.pol.mean[k], self.pol.log_prob[k],
                self.pol.values[k], t)
        else:
            policy_act(sim, slab.obs_in[k], self.blob, slab.actions[k], self.pol.mean[k], self.pol.log_prob[k], self.pol.values[k], t,
                       self.activation)
        if self.device_terms:
            sim.step_terms(slab.actions[k], t, out=self._step_outputs(k), log=self.logs[k], term_log=self.term_logs[k])
        else:
            sim.step(slab.actions[k], t, out=self._step_outputs(k), log=self.logs[k])
        sim.policy_observe(t, out=slab.obs[k])
        if self.critic:
            sim.critic_observe(out=slab.critic_obs_in[k + 1])

    def observe0(self, step_counter: int):
        """The first rollout row (observation_manager.compute at `step_counter`, call 0) into obs0 (and cobs0)."""
        self.sim.observe_policy_row(step_counter, 0, self.obs0)
        if self.critic:
            self.sim.critic_observe(out=self.cobs0)

    def _body(self):
        self.slab.obs_in[0].copy_(self.obs0)
        if self.critic:
            self.slab.critic_obs_in[0].copy_(self.cobs0)
        for k in range(self.T):
            t = WheeledSim.device_counter_plus(k)
            if self.table:
                self._table_step(k, t)
            elif self.critic:
                act = policy_act_wide_asym if self.activation == "relu" else policy_act_asym
                act(self.sim, self.slab.obs_in[k], self.slab.critic_obs_in[k], self.blob, self.slab.actions[k],
                    self.pol.mean[k], self.pol.log_prob[k], self.pol.values[k], t)
                self.sim.step(self.slab.actions[k], t, out=self.slab.step_outputs(k), log=self.logs[k])
                self.sim.critic_observe(out=self.slab.critic_obs_in[k + 1])
            elif self.deterministic:
                if self.activation == "relu" or self.rows:
                    actor_mean(self.blob, self.sim.obs_dim, self.slab.obs_in[k], self.activation, out=self.slab.actions[k])
                    self.sim.step(self.slab.actions[k], t, out=self.slab.step_outputs(k), log=self.logs[k])
                else:
                    act_infer_step(self.sim, self.slab.obs_in[k], self.blob, self.slab.actions[k], self.slab.step_outputs(k),
                                   self.logs[k], t)
            elif self.device_terms:
                policy_act(self.sim, self.slab.obs_in[k], self.blob, self.slab.actions[k], self.pol.mean[k], self.pol.log_prob[k],
                           self.pol.values[k], t, self.activation)
                self.sim.step_terms(self.slab.actions[k], t, out=self.slab.step_outputs(k), log=self.logs[k], term_log=self.term_logs[k])
            elif self.activation == "relu" or self.rows:
                policy_act(self.sim, self.slab.obs_in[k], self.blob, self.slab.actions[k], self.pol.mean[k], self.pol.log_prob[k],
                           self.pol.values[k], t, self.activation)
                self.sim.step(self.slab.actions[k], t, out=self.slab.step_outputs(k), log=self.logs[k])
            else:
                act_step(self.sim, self.slab.obs_in[k], self.blob, self.slab.actions[k], self.pol.mean[k], self.pol.log_prob[k],
                         self.pol.values[k], self.slab.step_outputs(k), self.logs[k], t)
        self.sim.advance_counter(self.T)
        self.obs0.copy_(self.slab.obs[self.T - 1])
        if self.critic:
            self.cobs0.copy_(self.slab.critic_obs_in[self.T])

    def capture(self, step_counter: int):
        sim = self.sim
        self.observe0(step_counter)
        sim.set_step_counter(step_counter)
        self.graph = torch.cuda.CUDAGraph()
        s = self._stream
        s.wait_stream(torch.cuda.current_stream(sim.device))
        with torch.cuda.stream(s):
            with torch.cuda.graph(self.graph, stream=s):
                self._body()
        torch.cuda.current_stream(sim.device).wait_stream(s)
        sim.set_step_counter(step_counter)       # (the captured advance_counter moved the HOST mirror; put both back)
        self._base = step_counter
        return self

    def run(self) -> RolloutSlab:
        self.graph.replay()
        self._base += self.T
        self.sim.note_device_counter(self._base)
        return self.slab


class StagedPolicyRollout:
    """The collection loop of an env with host-side Python reward / termination terms: T x (policy, then the env's staged step
    ``env.staged_step``: stage a -> Python terms -> stage b), issued eagerly because the terms are arbitrary torch code that
    may sync the host.  The policy is ``policy_act`` (wl_policy_act_elu for "elu", wl_policy_act for "relu") on the host's
    step counter, which the staged step advances by one per step.  The slab is filled as ``FusedPolicyRollout`` fills it
    (``obs_in[k]`` -> actions / mean / log-prob / values [k]; rewards, ``obs[k] = obs_in[k+1]``, terminated, truncated [k];
    ``logs[k]`` the episode-log row), and ``py_logs[k]`` [T, len(py_names)] f64 holds what env.step's ``extras["log"]`` has at
    step k for each Python term's key (``py_names``)."""

    def __init__(self, env, blob: torch.Tensor, T: int = 128, activation: str = "elu"):
        sim = env.sim
        if env._py_obs:
            raise NotImplementedError("Python observation terms widen the observation past the slab row the staged step writes")
        if (sim.num_envs * sim.obs_dim) % 2:
            raise ValueError("the slab's observation rows are written pair-wise: num_envs * obs_dim must be even")
        self.env, self.sim, self.blob, self.T, self.activation = env, sim, blob, T, check_activation(activation)
        self.slab = RolloutSlab(T, sim.num_envs, sim.obs_dim, 2, sim.device, policy_fields=True)
        self.logs = torch.zeros((T, 16), dtype=torch.float32, device=sim.device)
        self.py_names = env.python_log_names
        self.py_logs = torch.zeros((T, len(self.py_names)), dtype=torch.float64, device=sim.device)
        self.obs0 = torch.empty((sim.num_envs, sim.obs_dim), dtype=torch.float32, device=sim.device)   # carried to the next run
        self._bits = torch.empty(sim.num_envs, dtype=torch.uint8, device=sim.device)
        self._stream = torch.cuda.Stream(device=sim.device)

    def start(self, step_counter: int):
        """Prime obs0 with the observation at `step_counter` (the env's ``common_step_counter``)."""
        self.sim.observe(step_counter, 0, out=self.obs0)
        return self

    def run(self) -> RolloutSlab:
        env, sim, slab = self.env, self.sim, self.slab
        slab.obs_in[0].copy_(self.obs0)
        for k in range(self.T):
            policy_act(sim, slab.obs_in[k], self.blob, slab.actions[k], slab.mean[k], slab.log_prob[k], slab.values[k],
                       env.common_step_counter, self.activation)
            *_, extra = env.staged_step(slab.actions[k], rew=slab.rewards[k], term_bits=self._bits,
                                        out=(slab.obs[k], slab.terminated[k], slab.truncated[k]), log=self.logs[k])
            if self.py_names:
                torch.stack([extra[name].to(torch.float64) for name in self.py_names], out=self.py_logs[k])
        self.obs0.copy_(slab.obs[self.T - 1])
        return slab
