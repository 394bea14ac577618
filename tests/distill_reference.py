"""A torch restatement of rsl_rl's ``StudentTeacher`` and ``Distillation.update()`` (rsl-rl-lib 2.3) [UPSTREAM-RECALL], run
the rsl_rl way: eager autograd over the student, ``mse_loss`` summed over ``gradient_length`` stored steps, ``clip_grad_norm_``
when ``max_grad_norm`` is set, ``torch.optim.Adam(student.parameters())`` at a fixed learning rate, ``.item()`` for the
loss log.  The reference the fused update (``wl_distill_update``) is tested against; it runs in any dtype (fp64 as the
accuracy yardstick)."""
from __future__ import annotations

import torch
from torch import nn

from wheeledlab_b200.policy import actor_critic_state_dict


class TorchDistillation:
    """student: the actor of a blob laid out by blob_layout(obs_dim); teacher: the actor of blob_layout(teacher_obs_dim)."""

    def __init__(self, student_blob: torch.Tensor, obs_dim: int, cfg, activation: str = "elu", dtype=torch.float64,
                 teacher_blob: torch.Tensor | None = None, teacher_obs_dim: int | None = None):
        act = nn.ELU if activation == "elu" else nn.ReLU
        dev = student_blob.device
        mk = lambda nin: nn.Sequential(nn.Linear(nin, 64), act(), nn.Linear(64, 64), act(), nn.Linear(64, 2)).to(dev, dtype)
        self.student = mk(obs_dim)
        sd = {k: v.to(dtype) for k, v in actor_critic_state_dict(student_blob, obs_dim).items()}
        self._load(self.student, sd)
        self.std = nn.Parameter(sd["std"].clone())          # StudentTeacher's scalar std: not in the optimizer
        self.teacher = None
        if teacher_blob is not None:
            self.teacher = mk(teacher_obs_dim)
            self._load(self.teacher, {k: v.to(dtype) for k, v in actor_critic_state_dict(teacher_blob, teacher_obs_dim).items()})
        self.cfg, self.dtype = cfg, dtype
        self.optimizer = torch.optim.Adam(self.student.parameters(), lr=cfg.learning_rate)
        self.chunk_grads = []                                # the (unclipped) gradient of every Adam step, student order

    @staticmethod
    def _load(net, sd):
        with torch.no_grad():
            for k in (0, 2, 4):
                net[k].weight.copy_(sd[f"actor.{k}.weight"]); net[k].bias.copy_(sd[f"actor.{k}.bias"])

    def act_inference(self, obs):
        return self.student(obs)

    def evaluate(self, teacher_obs):
        with torch.no_grad():
            return self.teacher(teacher_obs)

    def update(self, obs: torch.Tensor, teacher_actions: torch.Tensor) -> dict:
        """obs [T, N, D], teacher_actions [T, N, 2]: Distillation.update() -- the epochs walk the T steps in order, the step
        count runs on across epochs, Adam steps after every gradient_length-th one; returns {"behavior": mean step loss} and
        keeps the per-step losses in ``self.losses``."""
        cfg = self.cfg
        obs, teacher_actions = obs.to(self.dtype), teacher_actions.to(self.dtype)
        loss, cnt, mean_loss = 0, 0, 0.0
        self.losses = []
        for _ in range(cfg.num_learning_epochs):
            for t in range(obs.shape[0]):
                behavior = nn.functional.mse_loss(self.act_inference(obs[t]), teacher_actions[t])
                loss = loss + behavior
                self.losses.append(behavior.item())
                mean_loss += behavior.item()
                cnt += 1
                if cnt % cfg.gradient_length == 0:
                    self.optimizer.zero_grad()
                    loss.backward()
                    self.chunk_grads.append([p.grad.detach().clone() for p in self.student.parameters()])
                    if cfg.max_grad_norm:
                        nn.utils.clip_grad_norm_(self.student.parameters(), cfg.max_grad_norm)
                    self.optimizer.step()
                    loss = 0
        return {"behavior": mean_loss / cnt}

    def state_dict(self) -> dict:
        return {f"actor.{k}": v for k, v in self.student.state_dict().items()}

    def adam_moments(self) -> dict:
        """{name: (exp_avg, exp_avg_sq)} of the student's parameters, actor.* names."""
        names = [f"actor.{k}.{w}" for k in (0, 2, 4) for w in ("weight", "bias")]
        st = self.optimizer.state
        return {n: (st[p]["exp_avg"], st[p]["exp_avg_sq"]) for n, p in zip(names, self.student.parameters()) if p in st}
