"""A torch restatement of rsl_rl ``PPO.update()`` (rsl-rl-lib >= 2.3.0) [UPSTREAM-RECALL] for the Drift-family actor-critic,
run the rsl_rl way: eager autograd, ``clip_grad_norm_``, ``torch.optim.Adam``, the KL-adaptive learning rate compared on
the host, ``.item()`` for the statistics.  The reference the fused update (``wl_ppo_update``) is tested and timed against;
it runs in any dtype (fp32 as rsl_rl, fp64 as the accuracy yardstick)."""
from __future__ import annotations

import torch
from torch import nn

from wheeledlab_b200.policy import actor_critic_state_dict


class TorchPPO:
    def __init__(self, blob: torch.Tensor, obs_dim: int, cfg, dtype=torch.float32):
        sd = {k: v.to(dtype) for k, v in actor_critic_state_dict(blob, obs_dim).items()}
        dev = blob.device
        mk = lambda out: nn.Sequential(nn.Linear(obs_dim, 64), nn.ELU(), nn.Linear(64, 64), nn.ELU(), nn.Linear(64, out)).to(dev, dtype)
        self.actor, self.critic = mk(2), mk(1)
        self.std = nn.Parameter(sd["std"].clone())
        with torch.no_grad():
            for name, net in (("actor", self.actor), ("critic", self.critic)):
                for k in (0, 2, 4):
                    net[k].weight.copy_(sd[f"{name}.{k}.weight"]); net[k].bias.copy_(sd[f"{name}.{k}.bias"])
        self.cfg, self.dtype, self.obs_dim = cfg, dtype, obs_dim
        self.learning_rate = cfg.learning_rate
        self.optimizer = torch.optim.Adam(self.parameters(), lr=cfg.learning_rate)
        self.trace = []                          # per mini-batch dict of what the branches / the lr rule saw

    def parameters(self):
        return list(self.actor.parameters()) + list(self.critic.parameters()) + [self.std]

    def state_dict(self) -> dict:
        sd = {f"actor.{k}": v for k, v in self.actor.state_dict().items()}
        sd.update({f"critic.{k}": v for k, v in self.critic.state_dict().items()})
        sd["std"] = self.std.detach()
        return sd

    def grads(self) -> dict:
        names = [f"actor.{k}.{w}" for k in (0, 2, 4) for w in ("weight", "bias")] + [f"critic.{k}.{w}" for k in (0, 2, 4) for w in ("weight", "bias")] + ["std"]
        return dict(zip(names, [p.grad.detach().clone() for p in self.parameters()]))

    def update(self, obs, actions, values, log_prob, mean, returns, advantages, perm, keep_grads=False):
        """Arguments flattened over [T*N] in slab order (cast to the reference dtype here); returns rsl_rl's statistics."""
        cfg, dt = self.cfg, self.dtype
        obs, actions, mean = obs.reshape(-1, self.obs_dim).to(dt), actions.reshape(-1, 2).to(dt), mean.reshape(-1, 2).to(dt)
        values, log_prob, returns = values.reshape(-1).to(dt), log_prob.reshape(-1).to(dt), returns.reshape(-1).to(dt)
        adv = advantages.reshape(-1).to(dt)
        adv = (adv - adv.mean()) / (adv.std() + 1e-8)
        old_sigma = self.std.detach().clone().expand_as(mean)
        n = obs.shape[0]
        B = n // cfg.num_mini_batches
        mv = ms = me = 0.0
        for _ in range(cfg.num_learning_epochs):
            for i in range(cfg.num_mini_batches):
                idx = perm[i * B:(i + 1) * B]
                o, a, v_old, lp_old, mu_old, R, A = obs[idx], actions[idx], values[idx], log_prob[idx], mean[idx], returns[idx], adv[idx]
                s_old = old_sigma[idx]
                mu = self.actor(o)
                sigma = self.std.expand_as(mu)
                dist = torch.distributions.Normal(mu, sigma, validate_args=False)
                lp = dist.log_prob(a).sum(dim=-1)
                value = self.critic(o).squeeze(-1)
                entropy = dist.entropy().sum(dim=-1)
                rec = {}
                with torch.inference_mode():
                    kl = torch.sum(torch.log(sigma / s_old + 1.0e-5) + (torch.square(s_old) + torch.square(mu_old - mu)) / (2.0 * torch.square(sigma)) - 0.5, dim=-1)
                    kl_mean = torch.mean(kl)
                    rec["kl"] = kl_mean.item()
                    if cfg.schedule == "adaptive":
                        if kl_mean > cfg.desired_kl * 2.0:
                            self.learning_rate = max(1e-5, self.learning_rate / 1.5)
                        elif kl_mean < cfg.desired_kl / 2.0 and kl_mean > 0.0:
                            self.learning_rate = min(1e-2, self.learning_rate * 1.5)
                        for g in self.optimizer.param_groups:
                            g["lr"] = self.learning_rate
                rec["lr"] = self.learning_rate
                ratio = torch.exp(lp - lp_old)
                surrogate = -A * ratio
                surrogate_clipped = -A * torch.clamp(ratio, 1.0 - cfg.clip_param, 1.0 + cfg.clip_param)
                surrogate_loss = torch.max(surrogate, surrogate_clipped).mean()
                if cfg.use_clipped_value_loss:
                    value_clipped = v_old + (value - v_old).clamp(-cfg.clip_param, cfg.clip_param)
                    value_losses = (value - R).pow(2)
                    value_losses_clipped = (value_clipped - R).pow(2)
                    value_loss = torch.max(value_losses, value_losses_clipped).mean()
                else:
                    value_loss = (R - value).pow(2).mean()
                loss = surrogate_loss + cfg.value_loss_coef * value_loss - cfg.entropy_coef * entropy.mean()
                self.optimizer.zero_grad()
                loss.backward()
                if keep_grads:
                    rec["grads"] = self.grads()
                    rec["ratio"], rec["A"] = ratio.detach(), A.detach()
                    rec["dv"] = (value - v_old).detach()
                    rec["vl"], rec["vlc"] = value_losses.detach() if cfg.use_clipped_value_loss else None, value_losses_clipped.detach() if cfg.use_clipped_value_loss else None
                rec["norm"] = nn.utils.clip_grad_norm_(self.parameters(), cfg.max_grad_norm).item()
                self.optimizer.step()
                rec["surrogate"], rec["value_function"], rec["entropy"] = surrogate_loss.item(), value_loss.item(), entropy.mean().item()
                mv += rec["value_function"]; ms += rec["surrogate"]; me += rec["entropy"]
                self.trace.append(rec)
        k = cfg.num_learning_epochs * cfg.num_mini_batches
        return {"value_function": mv / k, "surrogate": ms / k, "entropy": me / k, "learning_rate": self.learning_rate, "kl": self.trace[-1]["kl"]}

    def forward(self, obs):
        with torch.no_grad():
            o = obs.reshape(-1, self.obs_dim).to(self.dtype)
            return self.actor(o), self.critic(o).squeeze(-1)
