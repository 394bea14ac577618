"""ManagerBasedRLEnv-compatible environment backed by the fused CUDA step.

Mirrors the surface of ``isaaclab.envs:ManagerBasedRLEnv`` that the reference's callers touch
(SURVEY.md 8b): ``train_rl.py:70-116``, ``modified_rsl_rl_runner.py:46-109``,
``create_and_step_env.py:26-44`` and the term code in ``wheeledlab/envs/mdp`` /
``wheeledlab_tasks``.  Same names, same argument meaning, same error behaviour (exceptions; no
silent CPU path).  Step ordering follows SURVEY.md 3.3 (A..I).
"""
from __future__ import annotations

import math
from types import SimpleNamespace

import torch

from .sim import WheeledSim
from .tasks import TaskSpec, make_task


class _Box:
    """Minimal gymnasium.spaces.Box stand-in (callers assign .low/.high, train_rl.py:73-74)."""

    def __init__(self, low, high, shape, dtype=torch.float32):
        self.low, self.high, self.shape, self.dtype = low, high, tuple(shape), dtype

    def sample(self, generator=None, device="cpu"):
        return torch.randn(self.shape, generator=generator, device=device)


class _LazyLog(dict):
    """extras["log"]: keys are known up front, values are 0-dim views of the device row of that step; the views are only
    created when somebody reads them (the train loop appends the dict every step and reads it once per iteration,
    modified_rsl_rl_runner.py:95-98).  The row of step t is written by the next launch on the handle (no grid-wide sync in
    the step): reading the log of the most recent step publishes it first (wl_log_flush, a 32-thread kernel)."""

    def __init__(self, row: torch.Tensor, index: dict, extra: dict | None = None, env=None):
        super().__init__((k, None) for k in index)
        self._row, self._index = row, index
        self._env, self._step = env, (env.common_step_counter if env is not None else None)
        self._extra = extra or {}                # entries of host-side (Python) terms: already 0-dim device tensors
        for k in self._extra:
            dict.__setitem__(self, k, None)

    def _ready(self):
        # the row of step t is written by the next launch on the handle: if this is still the most recent step, flush now
        env = self._env
        if env is not None and env.common_step_counter == self._step:
            env.sim.flush_log()
        self._env = None

    def __getitem__(self, k):
        if k in self._extra:
            return self._extra[k]
        if self._env is not None:
            self._ready()
        return self._row[self._index[k]]

    def get(self, k, default=None):
        if k in self._extra:
            return self._extra[k]
        if k not in self._index:
            return default
        return self[k]

    def items(self):
        return [(k, self[k]) for k in list(self._index) + list(self._extra)]

    def values(self):
        return [self[k] for k in list(self._index) + list(self._extra)]


class RewardTermCfgView:
    """What reward_manager.get_term_cfg returns: an object with a mutable ``weight`` (curriculums.py:33-35)."""

    def __init__(self, name: str, weight: float):
        self.name, self.weight = name, weight
        self.params = {}


class RewardManager:
    def __init__(self, env):
        self._env = env
        self.active_terms = list(env.spec.reward_names)

    def _slot(self, name):
        try:
            return self.active_terms.index(name)
        except ValueError:
            raise ValueError(f"Reward term '{name}' not found.") from None

    def get_term_cfg(self, name) -> RewardTermCfgView:
        return RewardTermCfgView(name, float(self._env.sim.rew_weight[self._slot(name)].item()))

    def set_term_cfg(self, name, cfg) -> None:
        self._env.sim.rew_weight[self._slot(name)] = float(cfg.weight)

    @property
    def weights(self) -> torch.Tensor:
        return self._env.sim.rew_weight[: len(self.active_terms)]


class CommandManager:
    """command_manager.get_command("goal_pose") -> [N,4] (pos_b xyz, heading_b), UniformPose2dCommand layout."""

    def __init__(self, env):
        self._env = env

    def get_command(self, name):
        from .sim import G_CMDB
        g = self._env.sim.groups[G_CMDB]
        out = torch.zeros((self._env.num_envs, 4), device=self._env.device)
        out[:, 0:2] = g[:, 0:2]
        out[:, 3] = g[:, 2]
        return out


class TerminationManager:
    def __init__(self, env):
        self._env = env
        self.active_terms = [n for n, _ in env.spec.termination_names]
        self.terminated = torch.zeros(env.num_envs, dtype=torch.bool, device=env.device)
        self.time_outs = torch.zeros(env.num_envs, dtype=torch.bool, device=env.device)

    @property
    def dones(self):
        return self.terminated | self.time_outs

    def get_term(self, name):
        """The term's OWN mask for the last step (IsaacLab TerminationManager.get_term), not the union: from the per-term bits
        the step kernel writes when the task has more than one non-time-out term (Elevation: cart_out_of_bounds, stuck,
        rollover, at_goal); host-side (Python) terms keep their own masks."""
        env = self._env
        if name in getattr(env, "_py_term_masks", {}):
            return env._py_term_masks[name]
        for k, t in enumerate(getattr(env, "_dev_terms", ())):
            if t.name == name and t.role != 0:
                return ((env.sim.device_term_masks >> k) & 1).to(torch.bool)
        names = env.spec.termination_names
        for j, (n, is_to) in enumerate(names):
            if n == name:
                bits = getattr(env, "_term_bits_staged", None) if env._staged else getattr(env, "_term_bits", None)
                if bits is not None:
                    return ((bits >> j) & 1).to(torch.bool)
                others = [m for m, to in names if to == is_to]
                if len(others) == 1:                       # the only term of its kind: its mask is the union
                    return self.time_outs if is_to else self.terminated
                raise RuntimeError(f"termination term {name!r}: per-term masks are not being recorded for this env")
        raise ValueError(f"Termination term '{name}' not found.")


class ActionManager:
    def __init__(self, env):
        self._env = env
        self.total_action_dim = env.spec.action_dim

    @property
    def action(self):
        return self._env.sim.last_action

    @property
    def prev_action(self):
        return self._env.sim.prev_action


class ObservationManager:
    def __init__(self, env):
        self._env = env
        self.group_obs_dim = {"policy": (env.spec.obs_dim,)}
        self._calls = 0

    def compute(self):
        """Re-samples the observation noise, like the reference (SURVEY 3.4)."""
        env = self._env
        if env._policy_terms:                    # (the table's row only: the built-in row would be thrown away)
            obs = env.sim.policy_observe(env.common_step_counter, self._calls)
        else:
            obs = env.sim.observe(env.common_step_counter, self._calls)
        self._calls += 1
        return env._obs_groups(obs)


class _RobotData:
    def __init__(self, sim: WheeledSim):
        self._sim = sim

    root_pos_w = property(lambda s: s._sim.root_pos_w)
    root_quat_w = property(lambda s: s._sim.root_quat_w)
    root_lin_vel_w = property(lambda s: s._sim.root_lin_vel_w)
    root_ang_vel_w = property(lambda s: s._sim.root_ang_vel_w)
    root_link_ang_vel_w = property(lambda s: s._sim.root_ang_vel_w)

    @staticmethod
    def _rot_inv(q, v):
        w, xyz = q[:, 0:1], q[:, 1:4]
        t = 2.0 * torch.cross(xyz, v, dim=-1)
        return v - w * t + torch.cross(xyz, t, dim=-1)

    @property
    def root_lin_vel_b(self):
        return self._rot_inv(self.root_quat_w, self.root_lin_vel_w)

    @property
    def root_ang_vel_b(self):
        return self._rot_inv(self.root_quat_w, self.root_ang_vel_w)

    @property
    def joint_vel(self):
        n = self._sim.num_envs
        out = torch.zeros((n, 10), device=self._sim.device)
        out[:, 0:4] = self._sim.wheel_vel
        out[:, 4:6] = self._sim.steer_vel
        out[:, 6:10] = self._sim.suspension_state()[1]
        return out

    @property
    def joint_pos(self):
        n = self._sim.num_envs
        out = torch.zeros((n, 10), device=self._sim.device)     # wheel angles are not tracked (not needed by any term)
        out[:, 4:6] = self._sim.steer_pos
        out[:, 6:10] = self._sim.suspension_state()[0]
        return out


class _Robot:
    """Articulation stand-in for env.scene["robot"] (write_root_* used by events.py:132-133)."""

    def __init__(self, env):
        self._env = env
        self.data = _RobotData(env.sim)
        self.joint_names = list(env.spec.joint_names)

    def find_joints(self, name_keys, joint_subset=None, preserve_order=False):
        import re
        keys = [name_keys] if isinstance(name_keys, str) else list(name_keys)
        ids, names = [], []
        for i, jn in enumerate(self.joint_names):
            if any(re.fullmatch(k, jn) for k in keys):
                ids.append(i)
                names.append(jn)
        if not ids:
            raise ValueError(f"Not all regular expressions are matched! {keys} vs {self.joint_names}")
        return ids, names

    def write_root_pose_to_sim(self, root_pose, env_ids=None):
        sim = self._env.sim
        ids = slice(None) if env_ids is None else env_ids
        sim.root_pos_w[ids] = root_pose[:, 0:3]
        sim.root_quat_w[ids] = root_pose[:, 3:7]

    def write_root_velocity_to_sim(self, root_velocity, env_ids=None):
        sim = self._env.sim
        ids = slice(None) if env_ids is None else env_ids
        sim.root_lin_vel_w[ids] = root_velocity[:, 0:3]
        sim.root_ang_vel_w[ids] = root_velocity[:, 3:6]


class _Scene:
    def __init__(self, env):
        self._assets = {"robot": _Robot(env)}
        self.env_origins = torch.zeros((env.num_envs, 3), device=env.device)   # env_spacing = 0 (:373)
        self.num_envs = env.num_envs
        self.sensors = {}

    def __getitem__(self, key):
        return self._assets[key]


class ManagerBasedRLEnv:
    """Drop-in for ``isaaclab.envs.ManagerBasedRLEnv`` on the Drift/Elevation/Visual gym ids."""

    _RING = 512      # step() / step_host() output buffers are reused after this many steps (fewer when rows are wide, see _ring_len)
    _HOST_OBS_RING = 4   # pinned host observation buffers of step_host(host_obs=True)

    metadata = {"render_modes": [None, "human", "rgb_array"], "isaac_sim_version": "h100-native"}

    def __init__(self, cfg: TaskSpec | str = "Isaac-MushrDriftRL-v0", render_mode=None, device="cuda:0", **task_kw):
        self._task_spec: TaskSpec = make_task(cfg, **task_kw) if isinstance(cfg, str) else cfg
        self.cfg = SimpleNamespace(is_finite_horizon=False, seed=int(self.spec.cfg.seed), spec=self.spec)
        self.render_mode = render_mode
        self.device = str(torch.device(device))
        self.sim = WheeledSim(self.spec, device)     # (the elevation height-field travels in spec.heightfield)
        self.num_envs = self.sim.num_envs
        self.step_dt = self.spec.step_dt
        self.physics_dt = float(self.spec.cfg.sim_dt)
        self.max_episode_length_s = self.spec.episode_length_s
        self.max_episode_length = int(self.spec.cfg.max_episode_length)   # ceil(episode_length_s/(dt*decimation)) in doubles
        self.common_step_counter = 0
        self.extras = {}
        self.scene = _Scene(self)
        self.action_manager = ActionManager(self)
        self.observation_manager = ObservationManager(self)
        self.reward_manager = RewardManager(self)
        self.termination_manager = TerminationManager(self)
        self.command_manager = CommandManager(self)
        self.single_action_space = _Box(-math.inf, math.inf, (self.spec.action_dim,))
        self.action_space = _Box(-math.inf, math.inf, (self.num_envs, self.spec.action_dim))
        self.single_observation_space = {"policy": _Box(-math.inf, math.inf, (self.spec.obs_dim,))}
        self.observation_space = {"policy": _Box(-math.inf, math.inf, (self.num_envs, self.spec.obs_dim))}
        self.log_episode_info = True
        self._log_index = {"Episode_Reward/" + n: k for k, n in enumerate(self.spec.reward_names)}
        self._log_index.update({"Episode_Termination/" + n: 9 + j for j, (n, _) in enumerate(self.spec.termination_names)})
        self._ring_len = max(8, min(self._RING, (2 << 30) // max(1, 4 * self.num_envs * self.spec.obs_dim)))
        self._step_ring = None
        self._host_io = None
        self._pinned_ptrs = {}                   # data_ptr -> c_void_p of caller buffers known to be pinned [N,2] f32
        self._ring = None
        self.host_transport = "zero_copy"        # or "copy": staged H2D / D2H copies (wl_step_host)
        self.host_obs = False                    # step_host: True -> observations are returned in pinned host memory too
        self._host_obs_ring = None
        # host-side (Python) MDP terms: evaluated between the two halves of the staged step (see add_reward_term)
        self._py_rewards, self._py_terms, self._py_obs = [], [], []
        self._py_events = []                     # host-side event terms (add_event_term): run between stage b1 and stage b2
        self._event_fired = None                 # [interval terms, N] u8: wl_event_timers' fired bytes
        self._py_sums = {}
        self._dev_terms = []                     # device terms (add_device_reward_term): evaluated by wl_step_terms
        self._dev_events = []                    # device event terms (add_device_event_term): applied by wl_step_terms
        self._term_log_ring = None
        self._critic_terms = []                  # the critic observation group (set_critic_observation)
        self._policy_terms = []                  # a modified policy observation group (set_policy_observation)
        self._policy_ring = None
        self._row_terms = []                     # noise, clip and scale on the Elevation / Visual row (set_row_terms)
        for name, func, weight, params in self.spec.python_reward_terms:
            self.add_reward_term(name, func, weight, params)
        for name, func, time_out, params in self.spec.python_termination_terms:
            self.add_termination_term(name, func, time_out, params)
        # per-term termination masks (TerminationManager.get_term): recorded by the step kernel when a union is not enough
        self._term_bits = None
        if sum(1 for _, to in self.spec.termination_names if not to) > 1:
            import ctypes as C
            from ._lib import check, lib
            self._term_bits = torch.zeros(self.num_envs, dtype=torch.uint8, device=self.device)
            check(lib.wl_set_term_bits(self.sim._h, C.c_void_p(self._term_bits.data_ptr())), "wl_set_term_bits")
        for name, func, role, weight, params in self.spec.device_terms:
            if role == "reward":
                self.add_device_reward_term(name, func, weight, params)
            else:
                self.add_device_termination_term(name, func, role == "time_out", params)
        for name, func, mode, params, interval_range_s in self.spec.device_events:
            self.add_device_event_term(name, func, mode, interval_range_s, params)
        if self.spec.reset_events:
            self.sim.set_reset_events(**{name: True for name in self.spec.reset_events})
        if self.spec.critic_terms:
            self.set_critic_observation([(name, fn, {"clip": (-clip, clip)} if clip else {}) for name, fn, clip in self.spec.critic_terms])
        if self.spec.row_critic:
            self.set_critic_observation(self.spec.row_critic)
        if self.spec.policy_terms:
            self.set_policy_observation([(name, fn, {"noise": nz, "clip": cl, "scale": sc}) for name, fn, nz, cl, sc in self.spec.policy_terms])
        if self.spec.row_terms:
            self.set_row_terms([(name, fn, {"noise": nz, "clip": cl, "scale": sc}) for name, fn, nz, cl, sc in self.spec.row_terms])
        # event_manager.apply(mode="startup")
        self.sim.startup()
        self._needs_reset = True
        for name, func, mode, params, interval_range_s in self.spec.python_event_terms:
            self.add_event_term(name, func, mode, params, interval_range_s)

    # -- gym surface ---------------------------------------------------------------------------
    @property
    def spec(self) -> TaskSpec:
        """The task description (TaskSpec).  gymnasium's make() assigns ITS EnvSpec to `env.spec`: that one is kept as
        `gym_spec` so that the assignment cannot clobber the task description the env works from."""
        return self._task_spec

    @spec.setter
    def spec(self, value):
        if isinstance(value, TaskSpec):
            self._task_spec = value
        else:
            self.gym_spec = value

    @property
    def unwrapped(self):
        return self

    @property
    def episode_length_buf(self):
        return self.sim.episode_length_buf

    @episode_length_buf.setter
    def episode_length_buf(self, value):
        # modified_rsl_rl_runner.py:46-49 assigns a randint tensor
        self.sim.episode_length_buf.copy_(value.to(torch.int32))

    def seed(self, seed: int = -1) -> int:
        """ManagerBasedEnv.seed: re-key the counter-based generator for every draw from now on (resets, pushes, observation
        noise, commands).  What startup already sampled (DR scatter, the reference-pose table) is not re-drawn -- the reference
        seeds before construction (hydra.py:30 overrides cfg.seed with the agent seed; pass seed= to make()/the task for that)."""
        if seed is not None and seed >= 0:
            self.sim.set_seed(int(seed))
        return int(self.spec.cfg.seed)

    def close(self):
        self.sim.close()

    def render(self, recompute=False):
        """No viewport: the reference renders through Omniverse RTX (video recording only, train_rl.py --video); returns None."""
        return None

    def reset(self, seed=None, options=None, env_ids=None):
        """Reset every env (or those of `env_ids`: _reset_idx), then run the reset-mode event terms on them, then observe."""
        self.sim.reset(env_ids, self.common_step_counter)
        if env_ids is None:
            self._needs_reset = False
        self._reset_events(None if env_ids is None else torch.as_tensor(env_ids, device=self.device).to(torch.int64).reshape(-1))
        obs = self.observation_manager.compute()
        return obs, self.extras

    def get_observations(self):
        """RslRlVecEnvWrapper.get_observations (SURVEY 3.4)."""
        obs = self.observation_manager.compute()
        return obs["policy"], {"observations": obs}

    # -- the critic observation group (privileged.py, wl_critic_observe; DESIGN 6m) --------------------------------------------
    def set_critic_observation(self, terms):
        """Give the env a ``critic`` observation group next to ``policy``: `terms` is a list of (name, fn, params), `fn` a
        function of the critic library (``privileged.wheel_friction`` / ``base_mass`` / ``motor_damping``, or IsaacLab's
        ``root_pos_w``, ``root_euler_xyz``, ``base_lin_vel``, ``base_ang_vel``, ``last_action``, ``joint_vel``, ``joint_pos``
        by name) or its name, `params` optionally holding ``clip=(-c, c)``.  The row is their concatenation, noise-free,
        at most 32 floats, formed on the device.  From then on ``step`` / ``reset`` / ``get_observations`` put a fresh
        ``[N, Dc]`` tensor at ``extras["observations"]["critic"]`` (and in the returned observation dict) and
        ``observation_manager.group_obs_dim["critic"]`` is ``(Dc,)``; ``[]`` removes the group.  Drift family, and not
        together with host-side Python terms or device terms.

        On Elevation a list that opens with the policy row's six terms in row order (``goal_relative_xyz``,
        ``root_euler_xyz``, ``base_lin_vel``, ``base_ang_vel``, ``last_action``, ``world_height_map``) is a row critic
        (``sim.set_row_critic``, DESIGN 6s): those six with their own ``clip`` and ``scale`` -- no noise, and the map with a
        clip -- then terms of the critic library, 689..721 floats.  Any other list goes to the library path above."""
        from . import privileged, row_terms
        terms = [(t, t, {}) if isinstance(t, str) else tuple(t) + ({},) * (3 - len(t)) for t in terms]
        if terms and (self._py_rewards or self._py_terms or self._py_obs or self._py_events):
            raise NotImplementedError("a critic observation group together with host-side Python terms is not implemented")
        if terms and (self._dev_terms or self._dev_events):
            raise NotImplementedError("a critic observation group together with device terms is not implemented")
        fns = [fn if isinstance(fn, str) else getattr(fn, "__name__", "") for _, fn, _ in terms]
        row = tuple(fns[:6]) == row_terms.task_terms("elevation")
        table, head = [], []
        for k, (name, fn, params) in enumerate(terms):
            p = dict(params or {})
            if row and k < 6:
                head.append(row_terms.lower_critic_term(name, fn, p.pop("noise", None), p.pop("clip", None), p.pop("scale", None)))
            else:
                table.append(privileged.lower_term(name, fn, p, clip=p.pop("clip", None)))
        privileged.check_width(table)
        if row:
            dc = self.sim.set_row_critic(head, table)     # (refuses a task other than Elevation)
        else:
            dc = self.sim.set_critic_terms(table)     # (refuses a task outside the Drift family)
        self._critic_terms = terms
        if dc:
            self.observation_manager.group_obs_dim["critic"] = (dc,)
        else:
            self.observation_manager.group_obs_dim.pop("critic", None)
            self.extras.pop("observations", None)

    # -- a modified policy observation group (policy_obs.py, wl_policy_observe; DESIGN 6q) ------------------------------------
    def set_policy_observation(self, terms):
        """Replace the built-in ``policy`` row by the concatenation of `terms`, a list of (name, fn, params): `fn` a function
        of the policy library (IsaacLab's ``root_pos_w``, ``root_euler_xyz``, ``base_lin_vel``, ``base_ang_vel``,
        ``last_action``, ``joint_vel``, ``joint_pos``, ``projected_gravity`` by name, or ``privileged.wheel_friction`` /
        ``base_mass`` / ``motor_damping``) or its name; `params` may hold ``noise`` (an ``AdditiveGaussianNoiseCfg`` /
        ``AdditiveUniformNoiseCfg`` or ``("gaussian", mean, std)`` / ``("uniform", n_min, n_max)``, drawn when the config's
        enable_corruption is set), ``clip=(lo, hi)`` and ``scale`` (a number or one per float), applied in that order after
        the value, as IsaacLab's ObservationManager does; anything else in `params` goes to the function.  At most 32 floats,
        formed on the device.  From then on ``step`` / ``reset`` / ``get_observations`` return that row as ``"policy"`` and
        ``observation_manager.group_obs_dim["policy"]`` is ``(Dp,)``; ``[]`` restores the built-in row.  Drift family only;
        it combines with device terms, device events and a critic group, not with host-side Python terms."""
        from . import policy_obs
        terms = [(t, t, {}) if isinstance(t, str) else tuple(t) + ({},) * (3 - len(t)) for t in terms]
        if terms and (self._py_rewards or self._py_terms or self._py_obs or self._py_events):
            raise NotImplementedError("a policy observation table together with host-side Python terms is not implemented")
        table = []
        for name, fn, params in terms:
            p = dict(params or {})
            table.append(policy_obs.lower_term(name, fn, p, p.pop("noise", None), p.pop("clip", None), p.pop("scale", None)))
        policy_obs.check_width(table)
        dp = self.sim.set_policy_terms(table)    # (refuses a task outside the Drift family)
        self._policy_terms = terms
        self._policy_ring = None
        d = dp or self.spec.obs_dim
        self.observation_manager.group_obs_dim["policy"] = (d,)
        self.single_observation_space = {"policy": _Box(-math.inf, math.inf, (d,))}
        self.observation_space = {"policy": _Box(-math.inf, math.inf, (self.num_envs, d))}

    # -- noise, clip and scale on the Elevation / Visual row (row_terms.py, wl_set_row_terms; DESIGN 6r) ---------------------
    def set_row_terms(self, terms):
        """Noise, clip and scale on the built-in Elevation or Visual ``policy`` row: `terms` is a list of (name, fn, params),
        one per term of the row in its order (Elevation: ``goal_relative_xyz``, ``root_euler_xyz``, ``base_lin_vel``,
        ``base_ang_vel``, ``last_action``, ``world_height_map``; Visual after the camera term: ``base_lin_vel``,
        ``base_ang_vel``, ``last_action``), `fn` the function or its name; `params` may hold ``noise`` (an
        ``AdditiveGaussianNoiseCfg`` / ``AdditiveUniformNoiseCfg`` or ``("gaussian", mean, std)`` / ``("uniform", n_min,
        n_max)``, drawn when the config's enable_corruption is set), ``clip=(lo, hi)`` and ``scale``, applied in that order
        after the raw value, as IsaacLab's ObservationManager does.  A term without a clip is unclipped: the registered
        group's clips must be restated (``row_terms.registered``).  The row's width does not change.  A term list other
        than the row's own raises NotImplementedError; ``[]`` restores the built-in row.  Every path that writes the row
        (``step``, device terms and events, the staged step of host-side Python terms, ``reset`` / ``get_observations``,
        ``step_host``) writes the modified one."""
        from . import row_terms
        from .tasks import TASK_ELEVATION, TASK_VISUAL
        task = {TASK_ELEVATION: "elevation", TASK_VISUAL: "visual"}.get(self.spec.cfg.task, "drift")
        terms = [(t, t, {}) if isinstance(t, str) else tuple(t) + ({},) * (3 - len(t)) for t in terms]
        table = []
        for name, fn, params in terms:
            p = dict(params or {})
            table.append(row_terms.lower_term(name, fn, p.pop("noise", None), p.pop("clip", None), p.pop("scale", None)))
        if table:
            row_terms.check_order(task, [t[0] for t in table])
        self.sim.set_row_terms(table)
        self._row_terms = [(name,) + t for (name, _, _), t in zip(terms, table)]

    @property
    def row_terms(self) -> list:
        """The env's row terms as ``(name, row term, noise, clip, scale)`` (``TaskSpec.row_terms``' form); [] = none."""
        return list(self._row_terms)

    def _obs_groups(self, obs: torch.Tensor) -> dict:
        """The observation dict of the current state: ``policy`` and, with a critic group, a fresh ``critic`` row; the same
        dict is what ``extras["observations"]`` holds then (RslRlVecEnvWrapper's convention, read by the reference's runner)."""
        groups = {"policy": self._append_py_obs(obs)}
        if self._critic_terms:
            groups["critic"] = self.sim.critic_observe()
            self.extras["observations"] = groups
        return groups

    def _curriculum_fire_mask(self) -> int:
        """Counter conditions of increase_reward_weight_over_time (curriculums.py:23-35) -- the host-side restatement the
        golden-vector test checks; at run time the same conditions are evaluated on the device (log_finalize)."""
        c, L = self.common_step_counter, self.max_episode_length
        if c % L != 0:
            return 0
        mask = 0
        num_episodes = c // L
        for k, t in enumerate(self.spec.curriculum):
            num_increases = num_episodes // t.episodes_per_increase
            if num_increases > t.max_increases:
                continue
            if (num_episodes + 1) % t.episodes_per_increase == 0:
                mask |= 1 << k
        return mask

    # -- host-side (Python) MDP terms: the reference's extension mechanism -----------------------------------------
    def add_reward_term(self, name: str, func, weight: float, params: dict | None = None):
        """Register ``func(env, **params) -> [N]`` as a reward term (IsaacLab RewardTermCfg semantics: contributes
        func * weight * step_dt, accumulated per episode and logged as Episode_Reward/<name>).  It runs on the
        post-physics, PRE-reset state, exactly where ManagerBasedRLEnv.step calls the reward manager: the env switches
        to the staged step (wl_step_stage_a -> Python terms -> wl_step_stage_b)."""
        self._refuse_mixing()
        self._py_rewards.append(SimpleNamespace(name=name, func=func, weight=float(weight), params=dict(params or {})))
        self._py_sums[name] = torch.zeros(self.num_envs, dtype=torch.float32, device=self.device)
        self.reward_manager.python_terms = [t.name for t in self._py_rewards]

    def add_termination_term(self, name: str, func, time_out: bool = False, params: dict | None = None):
        """Register ``func(env, **params) -> [N] bool`` as a termination term (TerminationTermCfg semantics; evaluated
        before the rewards, OR-ed into terminated / time_outs, resets the env in the same step)."""
        self._refuse_mixing()
        self._py_terms.append(SimpleNamespace(name=name, func=func, time_out=bool(time_out), params=dict(params or {})))
        self.termination_manager.python_terms = [t.name for t in self._py_terms]

    def add_event_term(self, name: str, func, mode: str, params: dict | None = None, interval_range_s=None, is_global_time: bool = False,
                       min_step_count_between_reset: int = 0):
        """Register ``func(env, env_ids, **params)`` as an event term (IsaacLab EventTermCfg semantics, DESIGN 6o).
        ``"startup"``: called once, now (the env has started up), with env_ids None.  ``"reset"``: called with the sorted
        int64 device tensor of the envs a step auto-reset, when there are any, after the built-in reset events and before the
        observation; also from ``reset(env_ids)``.  ``"interval"``: per env, a timer drawn from ``interval_range_s`` = (lo, hi)
        counts down by step_dt; the function is called with the envs whose timer ran out (timers restart at reset), after the
        built-in pushes, in registration order.  Events write the state through ``scene["robot"].write_root_pose_to_sim`` /
        ``write_root_velocity_to_sim``, the ``data`` views and ``episode_length_buf``.  The env then steps through the staged
        step (stage a, b1, events, b2).  Refused by name: "prestartup" and other modes, is_global_time=True,
        min_step_count_between_reset != 0, more than 8 interval terms."""
        from .compat import MAX_INTERVAL_EVENTS, check_event_term
        check_event_term(name, mode, interval_range_s, is_global_time, min_step_count_between_reset)
        self._refuse_mixing()
        intervals = [t for t in self._py_events if t.mode == "interval"]
        if mode == "interval" and len(intervals) >= MAX_INTERVAL_EVENTS:
            raise NotImplementedError(f"event term {name}: more than {MAX_INTERVAL_EVENTS} Python interval event terms")
        term = SimpleNamespace(name=name, func=func, mode=mode, params=dict(params or {}),
                               interval_range_s=None if mode != "interval" else tuple(float(v) for v in interval_range_s))
        if mode == "startup":
            func(self, None, **term.params)
        elif mode == "interval":
            self.sim.set_event_timers([t.interval_range_s for t in intervals + [term]])
            self._event_fired = torch.zeros((len(intervals) + 1, self.num_envs), dtype=torch.uint8, device=self.device)
        self._py_events.append(term)

    def _reset_events(self, env_ids: torch.Tensor | None):
        """The reset-mode event terms on `env_ids` (None: every env), in registration order."""
        terms = [t for t in self._py_events if t.mode == "reset"]
        if terms and env_ids is None:
            env_ids = torch.arange(self.num_envs, dtype=torch.int64, device=self.device)
        for term in terms:
            term.func(self, env_ids, **term.params)

    @property
    def _staged(self) -> bool:
        """Whether env.step runs the staged step: host-side reward, termination or event terms."""
        return bool(self._py_rewards or self._py_terms or self._py_events)

    # -- device terms: the reference's unregistered reward / termination functions, in CUDA (device_terms.py) ---------------
    def _refuse_mixing(self, device: bool = False):
        if getattr(self, "_policy_terms", None) and not device:
            raise NotImplementedError("a policy observation table together with host-side Python terms is not implemented")
        if getattr(self, "_critic_terms", None):
            raise NotImplementedError("a critic observation group together with " + ("device terms" if device else "host-side Python terms")
                                      + " is not implemented")
        if (self._py_rewards or self._py_terms or getattr(self, "_py_events", None)) if device else \
                (self._dev_terms or getattr(self, "_dev_events", None)):
            raise NotImplementedError("an env runs either device terms or host-side Python reward / termination terms, not both")

    def _add_device_term(self, name, func, role, weight, params):
        from . import device_terms as dtm
        self._refuse_mixing(device=True)
        tk = dtm.lookup(func) if callable(func) else dtm.resolve(func)
        if tk is None:
            raise NotImplementedError(f"device term {name!r}: {getattr(func, '__module__', '?')}.{getattr(func, '__name__', func)} "
                                      "is not in the device-term library (register it with add_reward_term as a Python term)")
        if len(self._dev_terms) >= dtm.MAX_TERMS:
            raise ValueError(f"at most {dtm.MAX_TERMS} device terms per env")
        if any(t.name == name for t in self._dev_terms):
            raise ValueError(f"device term {name!r} is already registered")
        term = SimpleNamespace(name=name, kind=tk, role=role, weight=float(weight), params=dtm.param_values(tk, params))
        table = [(t.kind.kind, t.role, t.weight, t.params) for t in self._dev_terms + [term]]
        self.sim.set_device_terms(table)          # (refuses a map term off the Visual task; resets the terms' state)
        self._dev_terms.append(term)
        if self._term_bits is None:               # get_term of a built-in term: its own mask, not the union with the device terms
            import ctypes as C
            from ._lib import check, lib
            self._term_bits = torch.zeros(self.num_envs, dtype=torch.uint8, device=self.device)
            check(lib.wl_set_term_bits(self.sim._h, C.c_void_p(self._term_bits.data_ptr())), "wl_set_term_bits")

    def add_device_reward_term(self, name: str, func, weight: float, params: dict | None = None):
        """Register a library function (device_terms.REGISTRY: the reference function object, or a kind) as a reward
        term evaluated on the device: the same value, weighting, episode sums and Episode_Reward/<name> entry as
        add_reward_term would give it, inside env.step's launches (wl_step_terms) and capturable in a graph."""
        from .device_terms import ROLE_REWARD
        self._add_device_term(name, func, ROLE_REWARD, weight, params)

    def add_device_termination_term(self, name: str, func, time_out: bool = False, params: dict | None = None):
        """Register a library function as a termination term evaluated on the device (fires when its value is nonzero;
        time_out=True truncates instead of terminating); get_term(name) and Episode_Termination/<name> cover it."""
        from .device_terms import ROLE_TERMINATION, ROLE_TIME_OUT
        self._add_device_term(name, func, ROLE_TIME_OUT if time_out else ROLE_TERMINATION, 0.0, params)

    def add_device_event_term(self, name: str, func, mode: str, interval_range_s=None, params: dict | None = None):
        """Register an event function of the device event library (device_events.REGISTRY: IsaacLab's
        ``push_by_setting_velocity``) as an event term applied on the device, inside env.step's launches (wl_step_terms) and
        capturable in a graph (DESIGN 6p).  ``"reset"``: applied to the envs the step reset, after the reset and the
        built-in pushes.  ``"interval"``: per env, a timer drawn from ``interval_range_s`` = (lo, hi) counts down by
        step_dt, and the term applies where it ran out (timers restart at reset).  Terms apply in registration order, before
        the step's command and observation.  ``env.reset()`` does not apply them.  Refused by name: what add_event_term
        refuses, startup mode, a function the library does not have, a ninth term, host-side Python terms on the env."""
        from . import device_events as dev
        from .compat import check_event_term
        check_event_term(name, mode, interval_range_s)
        dev.check_mode(name, mode)
        if dev.lookup(func) is None:
            raise NotImplementedError(f"event term {name}: {getattr(func, '__module__', '?')}.{getattr(func, '__name__', func)} "
                                      "is not in the device event library (register it with add_event_term as a Python event term)")
        self._refuse_mixing(device=True)
        if len(self._dev_events) >= dev.MAX_TERMS:
            raise NotImplementedError(f"event term {name}: more than {dev.MAX_TERMS} device event terms")
        if any(t.name == name for t in self._dev_events):
            raise ValueError(f"device event term {name!r} is already registered")
        term = SimpleNamespace(name=name, func=func, mode=mode, ranges=dev.velocity_ranges(name, params),
                               interval_range_s=None if mode != "interval" else tuple(float(v) for v in interval_range_s))
        self.sim.set_device_events([(t.mode, t.interval_range_s, t.ranges) for t in self._dev_events + [term]])
        self._dev_events.append(term)

    @property
    def device_log_names(self) -> list:
        """The extras["log"] keys of the device terms, in table order (the order of wl_step_terms' term_log)."""
        from .device_terms import ROLE_REWARD
        return [("Episode_Reward/" if t.role == ROLE_REWARD else "Episode_Termination/") + t.name for t in self._dev_terms]

    def add_observation_term(self, name: str, func, params: dict | None = None):
        """Register ``func(env, **params) -> [N, k]``; appended to the policy observation (after the built-in terms)."""
        if self._policy_terms:
            raise NotImplementedError("a policy observation table together with host-side Python observation terms is not implemented")
        term = SimpleNamespace(name=name, func=func, params=dict(params or {}))
        k = int(func(self, **term.params).reshape(self.num_envs, -1).shape[1])
        self._py_obs.append(term)
        d = self.observation_manager.group_obs_dim["policy"][0] + k
        self.observation_manager.group_obs_dim["policy"] = (d,)
        self.single_observation_space = {"policy": _Box(-math.inf, math.inf, (d,))}
        self.observation_space = {"policy": _Box(-math.inf, math.inf, (self.num_envs, d))}

    def _append_py_obs(self, obs: torch.Tensor) -> torch.Tensor:
        if not self._py_obs:
            return obs
        return torch.cat([obs] + [t.func(self, **t.params).reshape(self.num_envs, -1).to(torch.float32) for t in self._py_obs], dim=1)

    def _step_staged(self, action: torch.Tensor):
        """env.step with Python terms in the loop: stage a (A-E) -> terminations -> rewards -> stage b (F-I)."""
        log = torch.empty(16, dtype=torch.float32, device=self.device) if self.log_episode_info else None
        obs, rew, terminated, truncated, extra = self.staged_step(action, log=log)
        if log is not None:
            self.extras["log"] = _LazyLog(log, self._log_index, extra, env=self)
        return {"policy": self._append_py_obs(obs)}, rew, terminated, truncated, self.extras

    def staged_step(self, action: torch.Tensor, rew: torch.Tensor | None = None, term_bits: torch.Tensor | None = None, out=None,
                    log: torch.Tensor | None = None):
        """One staged step at ``common_step_counter`` -- stage a, the Python termination terms, then the Python reward terms
        (func * weight * step_dt, weight 0 skipped, per-episode sums kept), stage b (with event terms: stage b1, the reset
        events, the interval timers and events, stage b2) -- into the caller's buffers where given:
        rew [N] f32, term_bits [N] u8, out = (obs [N, obs_dim] f32, terminated [N] u8, truncated [N] u8), log f32[16] (the
        episode-log row, written by the next launch on the handle).  Advances ``common_step_counter`` by one and sets the
        termination manager's masks.  Returns (obs, rew, terminated, truncated, extra): `extra` holds the Python terms'
        ``Episode_Reward/<name>`` / ``Episode_Termination/<name>`` entries as 0-dim device tensors when `log` is given,
        else None.  env.step and the runner's staged rollout both run their Python terms through this."""
        t = self.common_step_counter
        sim, tm = self.sim, self.termination_manager
        rew, bits = sim.step_stage_a(action, t, rew=rew, term_bits=term_bits)
        built_in_to = (bits & 1).bool()
        built_in_term = (bits & 0xFE).bool()
        self._term_bits_staged = bits            # per-term masks of the built-in terms (get_term)
        extra_term = extra_to = None
        fired = {}
        self._py_term_masks = fired
        for term in self._py_terms:
            v = term.func(self, **term.params).to(torch.bool)
            fired[term.name] = v
            if term.time_out:
                extra_to = v if extra_to is None else (extra_to | v)
            else:
                extra_term = v if extra_term is None else (extra_term | v)
        # what reward terms such as is_terminated_term see (TerminationManager.compute runs before RewardManager.compute)
        tm.terminated = built_in_term if extra_term is None else (built_in_term | extra_term)
        tm.time_outs = built_in_to if extra_to is None else (built_in_to | extra_to)
        for term in self._py_rewards:
            if term.weight == 0.0:
                continue
            val = term.func(self, **term.params).to(torch.float32) * (term.weight * self.step_dt)
            rew += val
            self._py_sums[term.name] += val
        if self._py_events:
            obs, term_u8, trunc_u8 = self._events_stage_b(bits, t, extra_term, extra_to, out, log)
        else:
            obs, term_u8, trunc_u8 = sim.step_stage_b(bits, t, extra_term, extra_to, out=out, log=log)
        self.common_step_counter = t + 1
        terminated, truncated = term_u8.view(torch.bool), trunc_u8.view(torch.bool)
        tm.terminated, tm.time_outs = terminated, truncated
        extra = None
        if log is not None:
            done = terminated | truncated
            cnt = done.sum().clamp(min=1).to(torch.float32)
            extra = {}
            for term in self._py_rewards:                        # RewardManager.reset: mean episodic sum / max_episode_length_s
                sums = self._py_sums[term.name]
                extra["Episode_Reward/" + term.name] = (sums * done).sum() / cnt / self.max_episode_length_s
                sums.masked_fill_(done, 0.0)
            for term in self._py_terms:
                extra["Episode_Termination/" + term.name] = (fired[term.name] & done).sum()
        return obs, rew, terminated, truncated, extra

    def _events_stage_b(self, bits, t, extra_term, extra_to, out, log):
        """Stage b with the event terms: b1 (log, auto-reset, built-in pushes), the reset events on the envs it reset, the
        interval timers and the interval events on the envs each one fired for, then b2 (commands, observation)."""
        sim, tm = self.sim, self.termination_manager
        obs_out, b1_out = (None, None) if out is None else (out[0], out[1:])
        term_u8, trunc_u8 = sim.step_stage_b1(bits, t, extra_term, extra_to, out=b1_out, log=log)
        tm.terminated, tm.time_outs = term_u8.view(torch.bool), trunc_u8.view(torch.bool)
        done = term_u8 | trunc_u8
        if any(e.mode == "reset" for e in self._py_events):
            ids = done.nonzero().squeeze(1)
            if ids.numel():
                self._reset_events(ids)
        if self._event_fired is not None:
            fired = sim.event_timers(done, t, self._event_fired)
            for k, term in enumerate(e for e in self._py_events if e.mode == "interval"):
                ids = fired[k].nonzero().squeeze(1)
                if ids.numel():
                    term.func(self, ids, **term.params)
        return sim.step_stage_b2(t, out=obs_out), term_u8, trunc_u8

    @property
    def python_log_names(self) -> list:
        """The extras["log"] keys of the Python reward and termination terms, in the order staged_step's `extra` has them."""
        return ["Episode_Reward/" + t.name for t in self._py_rewards] + ["Episode_Termination/" + t.name for t in self._py_terms]

    def step(self, action: torch.Tensor):
        if self._needs_reset:
            self.reset()
        if action.dtype != torch.float32 or not action.is_contiguous() or str(action.device) != self.device:
            action = action.to(self.device, torch.float32).contiguous()
        if self._staged:
            return self._step_staged(action)
        t = self.common_step_counter
        # outputs live in a ring of preallocated buffers (no allocator call per step; a returned tensor stays valid for
        # _ring_len steps -- rsl_rl copies into its storage at once, play_policy.py keeps at most one episode of references)
        if self._step_ring is None:
            n, dev = self.num_envs, self.device
            self._step_ring = [((torch.empty((n, self.spec.obs_dim), dtype=torch.float32, device=dev), torch.empty(n, dtype=torch.float32, device=dev),
                                 torch.empty(n, dtype=torch.uint8, device=dev), torch.empty(n, dtype=torch.uint8, device=dev)),
                                torch.empty(16, dtype=torch.float32, device=dev)) for _ in range(self._ring_len)]
        out, log = self._step_ring[t % self._ring_len]
        if not self.log_episode_info:
            log = None
        if self._dev_terms or self._dev_events:
            if self._term_log_ring is None:
                self._term_log_ring = torch.zeros((self._ring_len, 8), dtype=torch.float32, device=self.device)
            term_log = self._term_log_ring[t % self._ring_len] if log is not None else None
            obs, rew, term_u8, trunc_u8 = self.sim.step_terms(action, t, out=out, log=log, term_log=term_log)
        else:
            obs, rew, term_u8, trunc_u8 = self.sim.step(action, t, out=out, log=log)
        if self._policy_terms:                   # the built-in row above is scratch; the table's row is the observation
            if self._policy_ring is None:
                self._policy_ring = torch.empty((self._ring_len, self.num_envs, self.sim.policy_obs_dim), dtype=torch.float32,
                                                device=self.device)
            obs = self.sim.policy_observe(t, out=self._policy_ring[t % self._ring_len])
        self.common_step_counter = t + 1
        # curriculum: applied by the step kernel's last CTA (uses the incremented counter and fires only if >= 1 env
        # reset, like the reference's call from _reset_idx) -- no host logic, no sync
        terminated, truncated = term_u8.view(torch.bool), trunc_u8.view(torch.bool)
        tm = self.termination_manager
        tm.terminated, tm.time_outs = terminated, truncated
        if log is not None:
            self.extras["log"] = self._episode_log(log, term_log if self._dev_terms else None)
        return self._obs_groups(obs), rew, terminated, truncated, self.extras

    def _episode_log(self, log: torch.Tensor, term_log: torch.Tensor | None = None):
        """extras["log"] (RewardManager/TerminationManager.reset, SURVEY Appendix B): lazy views of the row the step
        kernel's last CTA wrote -- device tensors, no extra launches, no host sync.  The device terms' entries are views
        of the term_log row wl_step_terms wrote."""
        extra = None if term_log is None else {k: term_log[j] for j, k in enumerate(self.device_log_names)}
        return _LazyLog(log, self._log_index, extra, env=self)

    def step_host(self, action_host: torch.Tensor):
        """env.step() for a HOST-side caller: `action_host` is a CPU tensor [N,2] (pinned for best speed).  One C call
        does H2D(actions) -> fused step -> D2H(reward, terminated, truncated) -> sync.  Returns
        (obs_dict [device], rew [pinned host], terminated [pinned host], truncated [pinned host], extras); the host
        result views are overwritten by the next step_host call.  With ``env.host_obs = True`` the observations are returned in
        pinned HOST memory as well (a ring of _RING buffers): D2H copy after the step (transport "copy") or written by the
        kernel over PCIe (transport "zero_copy")."""
        if self._py_rewards or self._py_terms or getattr(self, "_py_events", None) or self._dev_terms or getattr(self, "_dev_events", None):
            raise NotImplementedError("step_host: Python and device terms need the staged step (use env.step)")
        if self._policy_terms:
            raise NotImplementedError("step_host: a policy observation table's row is formed by a second kernel (use env.step)")
        if self._needs_reset:
            self.reset()
        if self._host_io is None:
            self._host_io = self.sim.make_host_io()
        io = self._host_io
        # a pinned, contiguous f32 block of the caller is read in place (DMA / PCIe reads straight from it); anything else is
        # staged through the env's own pinned buffer
        ptr = action_host.data_ptr()
        if ptr == io["h_action"].data_ptr():
            p_action = None
        elif (action_host.dtype == torch.float32 and action_host.is_contiguous() and action_host.shape == (self.num_envs, 2)
              and action_host.is_pinned()):                  # (queried every call: an address may be reused by pageable memory)
            p_action = self._pinned_ptrs.get(ptr)
            if p_action is None:
                import ctypes as C
                if len(self._pinned_ptrs) > 65536:
                    self._pinned_ptrs.clear()
                p_action = self._pinned_ptrs[ptr] = C.c_void_p(ptr)
        else:
            p_action = None
            io["h_action"].copy_(action_host)
        t = self.common_step_counter
        # outputs come from a ring of preallocated device buffers (valid for _RING steps, like IsaacLab's own reuse)
        k = t % self._ring_len
        if self._ring is None:
            import ctypes as C
            self._ring = []
            for _ in range(self._ring_len):
                o = torch.empty((self.num_envs, self.spec.obs_dim), dtype=torch.float32, device=self.device)
                lg = torch.empty(16, dtype=torch.float32, device=self.device)
                self._ring.append((o, lg, C.c_void_p(o.data_ptr()), C.c_void_p(lg.data_ptr()), _LazyLog(lg, self._log_index)))
        obs, log, p_obs, p_log, lazy = self._ring[k]
        if not self.log_episode_info:
            log, p_log = None, None
        h_obs = None
        if self.host_obs:                                # the caller lives on the host: observations come back too
            if self._host_obs_ring is None:
                self._host_obs_ring = [torch.empty((self.num_envs, self.spec.obs_dim), dtype=torch.float32).pin_memory()
                                       for _ in range(self._HOST_OBS_RING)]
            h_obs = self._host_obs_ring[t % self._HOST_OBS_RING]
        if self.host_transport == "zero_copy":
            if h_obs is not None:                        # the kernel writes the observation rows straight into pinned host memory
                import ctypes as C
                self.sim.step_host_zero_copy(io, t, h_obs, log, C.c_void_p(h_obs.data_ptr()), p_log, p_action)
            else:
                self.sim.step_host_zero_copy(io, t, obs, log, p_obs, p_log, p_action)
        else:
            self.sim.step_host(io, t, obs, log, h_obs=h_obs, p_action=p_action)
        if h_obs is not None:
            obs = h_obs
        self.common_step_counter = t + 1
        tm = self.termination_manager
        tm.terminated, tm.time_outs = io["terminated"], io["truncated"]
        if log is not None:
            lazy._env, lazy._step = self, t + 1          # one lazy view per ring slot (its row tensor never changes)
            self.extras["log"] = lazy
        return {"policy": obs}, io["rew"], io["terminated"], io["truncated"], self.extras

    @property
    def host_action_buffer(self) -> torch.Tensor:
        """Pinned [N,2] buffer a host-side policy can write actions into (zero-copy input of step_host)."""
        if self._host_io is None:
            self._host_io = self.sim.make_host_io()
        return self._host_io["h_action"]


def make(task_id: str, cfg=None, render_mode=None, device="cuda:0", device_terms: bool = False, allow_python_terms: bool = False,
         **kw) -> ManagerBasedRLEnv:
    """gym.make(<id>, cfg=...) equivalent for the registered WheeledLab ids.  `cfg` may also be a reference env-cfg object,
    lowered by compat.spec_from_reference_cfg with `device_terms` / `allow_python_terms`."""
    if cfg is not None and not isinstance(cfg, (str, TaskSpec)):
        from .compat import spec_from_reference_cfg
        cfg = spec_from_reference_cfg(cfg, allow_python_terms=allow_python_terms, device_terms=device_terms)
    return ManagerBasedRLEnv(cfg if cfg is not None else task_id, render_mode=render_mode, device=device, **kw)
