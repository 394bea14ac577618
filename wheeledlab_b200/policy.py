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

from ._lib import WlPolicyOut, check, lib
from .distributed import RolloutSlab
from .sim import WheeledSim, _stream_ptr

HIDDEN = 64


def blob_layout(obs_dim: int):
    off = (C.c_int32 * 13)()
    total = lib.wl_policy_blob_floats(obs_dim, off)
    return list(off), total


def _linears(net):
    ls = [m for m in net.modules() if isinstance(m, torch.nn.Linear)]
    if len(ls) != 3 or ls[0].out_features != HIDDEN or ls[1].in_features != HIDDEN or ls[1].out_features != HIDDEN:
        raise NotImplementedError("wl_act_step implements the reference's [64, 64] ELU actor / critic only")
    return ls


def pack_actor_critic(actor, critic, std: torch.Tensor, obs_dim: int, device, out: torch.Tensor | None = None) -> torch.Tensor:
    """actor / critic: torch modules holding three nn.Linear (obs->64->64->2 / ->1, ELU in between); std: [2].
    Returns (or refills, when `out` is given -- e.g. after an optimiser step) the fp32 device blob wl_act_step reads."""
    off, total = blob_layout(obs_dim)
    blob = out if out is not None else torch.zeros(total, dtype=torch.float32, device=device)
    with torch.no_grad():
        for net_i, (net, nout) in enumerate(((actor, 2), (critic, 1))):
            ls = _linears(net)
            if ls[0].in_features != obs_dim or ls[2].out_features != nout:
                raise ValueError("network shape does not match the task")
            for k, lin in enumerate(ls):
                wt = lin.weight.detach().to(device=device, dtype=torch.float32).t().contiguous().reshape(-1)   # input-major
                o = off[net_i * 6 + 2 * k]
                blob[o:o + wt.numel()].copy_(wt)
                o = off[net_i * 6 + 2 * k + 1]
                blob[o:o + lin.bias.numel()].copy_(lin.bias.detach().to(device=device, dtype=torch.float32))
        blob[off[12]:off[12] + 2].copy_(std.detach().to(device=device, dtype=torch.float32))
    return blob


def _blob_layers(blob: torch.Tensor, obs_dim: int):
    """Zero-copy views of the blob: per net, three (W [in, out] input-major, b [out]) pairs; plus std [2]."""
    off, _ = blob_layout(obs_dim)
    nets = []
    for net_i, nout in enumerate((2, 1)):
        o = off[net_i * 6:net_i * 6 + 6]
        nets.append([(blob[o[0]:o[0] + obs_dim * HIDDEN].view(obs_dim, HIDDEN), blob[o[1]:o[1] + HIDDEN]),
                     (blob[o[2]:o[2] + HIDDEN * HIDDEN].view(HIDDEN, HIDDEN), blob[o[3]:o[3] + HIDDEN]),
                     (blob[o[4]:o[4] + HIDDEN * nout].view(HIDDEN, nout), blob[o[5]:o[5] + nout])])
    return nets[0], nets[1], blob[off[12]:off[12] + 2]


def actor_critic_state_dict(blob: torch.Tensor, obs_dim: int) -> dict:
    """The blob as an rsl_rl ActorCritic state dict (actor.0/2/4.weight|bias, critic.0/2/4.weight|bias, std) [UPSTREAM-RECALL]:
    the ``model_state_dict`` of the checkpoints rsl_rl's runner saves and ``play_policy.py`` loads.  Tensors are copies."""
    actor, critic, std = _blob_layers(blob, obs_dim)
    sd = {}
    for name, layers in (("actor", actor), ("critic", critic)):
        for k, (w, b) in enumerate(layers):
            sd[f"{name}.{2 * k}.weight"] = w.t().contiguous()
            sd[f"{name}.{2 * k}.bias"] = b.clone()
    sd["std"] = std.clone()
    return sd


def load_actor_critic_state_dict(sd: dict, obs_dim: int, out: torch.Tensor | None = None, device=None) -> torch.Tensor:
    """Inverse of actor_critic_state_dict: fills `out` (or a new zeroed blob) from an rsl_rl ActorCritic state dict."""
    if out is None:
        out = torch.zeros(blob_layout(obs_dim)[1], dtype=torch.float32, device=device or sd["std"].device)
    actor, critic, std = _blob_layers(out, obs_dim)
    with torch.no_grad():
        for name, layers in (("actor", actor), ("critic", critic)):
            for k, (w, b) in enumerate(layers):
                wt, bt = sd[f"{name}.{2 * k}.weight"], sd[f"{name}.{2 * k}.bias"]
                if tuple(wt.shape) != (w.shape[1], w.shape[0]) or tuple(bt.shape) != tuple(b.shape):
                    raise ValueError(f"{name}.{2 * k}: shape {tuple(wt.shape)} does not match the [64, 64] ELU network of obs_dim {obs_dim}")
                w.copy_(wt.t())
                b.copy_(bt)
        std.copy_(sd["std"])
    return out


ACTIVATIONS = {"elu": torch.nn.functional.elu, "relu": torch.nn.functional.relu}


def check_activation(activation: str) -> str:
    if activation not in ACTIVATIONS:
        raise ValueError(f"activation must be 'elu' (the Drift family's network) or 'relu' (Elevation / Visual), not {activation!r}")
    return activation


def critic_value(blob: torch.Tensor, obs_dim: int, obs: torch.Tensor, activation: str = "elu") -> torch.Tensor:
    """V(obs) [N] in torch from zero-copy views of the blob (the bootstrap value of compute_returns): a CUDA graph that
    captures it reads the weights the last update left in the blob."""
    act = ACTIVATIONS[check_activation(activation)]
    _, critic, _ = _blob_layers(blob, obs_dim)
    x = obs
    for k, (w, b) in enumerate(critic):
        x = torch.addmm(b, x, w)
        if k < 2:
            x = act(x)
    return x.squeeze(-1)


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


def policy_act(sim: WheeledSim, obs_in: torch.Tensor, blob: torch.Tensor, actions: torch.Tensor, mean: torch.Tensor,
               log_prob: torch.Tensor, value: torch.Tensor, step_counter: int):
    """One launch (wl_policy_act): value / mean / sample / log-prob of `obs_in` [N, obs_dim] under the ReLU network in `blob`,
    for any obs_dim up to 4096.  The env is not stepped: follow with sim.step(actions, step_counter)."""
    po = WlPolicyOut(actions.data_ptr(), mean.data_ptr(), log_prob.data_ptr(), value.data_ptr())
    check(lib.wl_policy_act(sim._h, C.c_void_p(obs_in.data_ptr()), C.c_void_p(blob.data_ptr()), po, step_counter,
                            _stream_ptr(sim.device)), "wl_policy_act")


class FusedPolicyRollout:
    """T policy-and-step launches captured as ONE CUDA graph: the reference's whole collection loop
    (modified_rsl_rl_runner.py:70-109).  activation "elu" (the Drift family): T x wl_act_step, the policy fused into the
    step; "relu" (Elevation, Visual): T x (wl_policy_act, then wl_step).  The blob is read at replay time, so refilling it
    in place (pack_actor_critic(..., out=blob)) after each PPO update needs no re-capture."""

    def __init__(self, sim: WheeledSim, blob: torch.Tensor, T: int = 128, slab: RolloutSlab | None = None, activation: str = "elu"):
        self.sim, self.blob, self.T, self.activation = sim, blob, T, check_activation(activation)
        if activation == "relu" and (sim.num_envs * sim.obs_dim) % 2:
            raise ValueError("wl_step writes each slab observation row pair-wise: num_envs * obs_dim must be even")
        self.slab = slab or RolloutSlab(T, sim.num_envs, sim.obs_dim, 2, sim.device, policy_fields=True)
        # values / log-prob / mean go straight into the slab (= the all-gather send buffer) when it has those fields
        self.pol = (SimpleNamespace(values=self.slab.values, log_prob=self.slab.log_prob, mean=self.slab.mean)
                    if hasattr(self.slab, "values") else PolicyBuffers(T, sim.num_envs, sim.device))
        self.logs = torch.zeros((T, 16), dtype=torch.float32, device=sim.device)
        # slab.obs_in[k] = the observation actions[k] / log_prob[k] / values[k] / mean[k] were computed from (rsl_rl
        # RolloutStorage.observations[k]); slab.obs[k] = obs_in[k+1] = what step k returned
        self.obs0 = torch.empty((sim.num_envs, sim.obs_dim), dtype=torch.float32, device=sim.device)    # carried to the next replay
        self.graph = None
        self._base = 0
        self._stream = torch.cuda.Stream(device=sim.device)

    def _body(self):
        self.slab.obs_in[0].copy_(self.obs0)
        for k in range(self.T):
            t = WheeledSim.device_counter_plus(k)
            if self.activation == "relu":
                policy_act(self.sim, self.slab.obs_in[k], self.blob, self.slab.actions[k], self.pol.mean[k], self.pol.log_prob[k],
                           self.pol.values[k], t)
                self.sim.step(self.slab.actions[k], t, out=self.slab.step_outputs(k), log=self.logs[k])
            else:
                act_step(self.sim, self.slab.obs_in[k], self.blob, self.slab.actions[k], self.pol.mean[k], self.pol.log_prob[k],
                         self.pol.values[k], self.slab.step_outputs(k), self.logs[k], t)
        self.sim.advance_counter(self.T)
        self.obs0.copy_(self.slab.obs[self.T - 1])

    def capture(self, step_counter: int):
        sim = self.sim
        sim.observe(step_counter, 0, out=self.obs0)
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
