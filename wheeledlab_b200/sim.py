"""WheeledSim: thin, allocation-owning wrapper over the C-ABI (one handle = one GPU's env shard).

torch is used for device memory and streams only; every computation is a launch of the
hand-written sm_90a kernels in ``csrc/`` through ``libwheeledlab_b200.so``.
"""
from __future__ import annotations

import ctypes as C

import torch

from . import _lib
from ._lib import WlConfig, check, lib
from .tasks import TaskSpec

# state groups (include/wheeledlab_b200.h)
G_POS, G_QUAT, G_LINVEL, G_ANGVEL, G_WHEEL, G_STEER, G_ACTION, G_SUM0, G_SUM1 = range(9)
G_PMASS, G_PMU_D, G_PMU_C, G_PKD, G_CMD, G_CMDB, G_PIW = 9, 10, 11, 12, 13, 14, 15
NUM_GROUPS = 16


_raw_stream = getattr(torch._C, "_cuda_getCurrentRawStream", None)     # cudaStream_t as an int, cheaper than building a Stream object


def _stream_ptr(device) -> C.c_void_p:
    """The CURRENT torch stream of `device` as a cudaStream_t (looked up every call: it follows torch.cuda.stream())."""
    if _raw_stream is not None:
        idx = device.index if isinstance(device, torch.device) else torch.device(device).index
        return C.c_void_p(_raw_stream(idx if idx is not None else torch.cuda.current_device()))
    return C.c_void_p(torch.cuda.current_stream(device).cuda_stream)


def upload_graph(graph: "torch.cuda.CUDAGraph", stream=None):
    """Upload an instantiated CUDA graph to the device now (set-up time) instead of inside its first replay (wl_graph_upload)."""
    st = stream if stream is not None else torch.cuda.current_stream()
    check(lib.wl_graph_upload(C.c_void_p(int(graph.raw_cuda_graph_exec())), C.c_void_p(st.cuda_stream)), "wl_graph_upload")


def _policy_term_array(terms, library: dict, what: str):
    """``[(name, noise, clip, scale)]`` (a bare name: none of them) -> (the normalised list, a wl_policy_term array)."""
    terms = [(t, None, None, None) if isinstance(t, str) else tuple(t) + (None,) * (4 - len(t)) for t in terms]
    arr = (_lib.WlPolicyTerm * max(1, len(terms)))()
    for k, (name, noise, clip, scale) in enumerate(terms):
        if name not in library:
            raise ValueError(f"{what} {name!r} is not in the library {sorted(library)}")
        if noise is not None and noise[0] not in _lib.WL_NOISE:
            raise ValueError(f"{what} {name!r}: unknown noise model {noise[0]!r}")
        d = arr[k]
        d.kind = library[name][0]
        if noise is not None:
            d.noise = _lib.WL_NOISE[noise[0]]
            d.noise_params[0], d.noise_params[1] = float(noise[1]), float(noise[2])
        if clip is not None:
            d.clip = 1
            d.clip_range[0], d.clip_range[1] = float(clip[0]), float(clip[1])
        if scale is not None:
            scale = (float(scale),) if isinstance(scale, (int, float)) else tuple(float(s) for s in scale)
            d.n_scale = len(scale)
            for j, s in enumerate(scale[:4]):
                d.scale[j] = s
    return terms, arr


def _device_u8_view(ptr: int, n: int, device) -> torch.Tensor:
    """uint8 [n] tensor over device memory the library owns (through __cuda_array_interface__; torch does not own it)."""
    class _Arr:
        __cuda_array_interface__ = {"shape": (n,), "typestr": "|u1", "data": (int(ptr), False), "version": 3}
    with torch.cuda.device(device):
        return torch.as_tensor(_Arr(), device=device)


class WheeledSim:
    def __init__(self, spec: TaskSpec, device: str | torch.device = "cuda:0", heightfield: torch.Tensor | None = None):
        self.spec = spec
        self.cfg: WlConfig = spec.cfg
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise _lib.WlError("wheeledlab_b200 runs on CUDA devices only (no CPU fallback)")
        if not torch.cuda.is_available():
            raise _lib.WlError("no CUDA device visible: wheeledlab_b200 has no CPU fallback")
        self.num_envs = int(self.cfg.num_envs)
        nbytes = lib.wl_state_bytes(self.num_envs)
        with torch.cuda.device(self.device):
            self._buf = torch.zeros(nbytes // 4, dtype=torch.float32, device=self.device)
            assert self._buf.data_ptr() % 256 == 0
            self._hf = None
            hf_ptr = None
            if heightfield is None and getattr(spec, "heightfield", None) is not None:
                heightfield = torch.from_numpy(spec.heightfield)
            if heightfield is not None:
                if heightfield.dtype == torch.uint8:                  # visual: raw aux blob
                    self._hf = heightfield.to(self.device).contiguous()
                else:
                    self._hf = heightfield.to(self.device, torch.float32).contiguous()
                hf_ptr = C.c_void_p(self._hf.data_ptr())
            handle = C.c_void_p()
            check(lib.wl_create(C.byref(self.cfg), C.c_void_p(self._buf.data_ptr()), nbytes, hf_ptr, C.byref(handle)),
                  "wl_create")
        self._h = handle
        n = self.num_envs
        self.groups = self._buf[: NUM_GROUPS * n * 4].view(NUM_GROUPS, n, 4)
        goff = lib.wl_globals_offset(n) // 4
        self._globals = self._buf[goff: goff + C.sizeof(_lib.WlGlobals) // 4]
        self.obs_dim = int(lib.wl_obs_dim(self._h))

    # -- lifetime ------------------------------------------------------------------
    def close(self):
        if getattr(self, "_h", None):
            lib.wl_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # -- hot path --------------------------------------------------------------------
    def startup(self):
        with torch.cuda.device(self.device):
            check(lib.wl_startup(self._h, _stream_ptr(self.device)), "wl_startup")

    def reset(self, env_ids: torch.Tensor | None, step_counter: int):
        with torch.cuda.device(self.device):
            if env_ids is None:
                check(lib.wl_reset(self._h, None, 0, step_counter, _stream_ptr(self.device)), "wl_reset")
            else:
                ids = env_ids.to(self.device, torch.int64).contiguous()
                check(lib.wl_reset(self._h, C.c_void_p(ids.data_ptr()), ids.numel(), step_counter,
                                   _stream_ptr(self.device)), "wl_reset")

    DEVICE_COUNTER = -1

    def set_seed(self, seed: int):
        """Re-key the counter-based generator (ManagerBasedEnv.seed); applies to every launch from now on."""
        check(lib.wl_set_seed(self._h, seed), "wl_set_seed")
        self.cfg.seed = seed

    @staticmethod
    def device_counter_plus(k: int) -> int:
        """step_counter value meaning "the counter base kept in device memory + k" (WL_DEVICE_COUNTER_PLUS)."""
        return -1 - k

    @property
    def handle(self) -> int:
        """The wl_sim* as an int (what torch.ops.wheeledlab_b200.* and foreign callers of the C-ABI take)."""
        return int(self._h.value)

    def set_peer_fanout(self, byte_deltas):
        """Every output row of step() is also stored at pointer + delta for each delta (peer symmetric buffers, see
        distributed.SymmetricRolloutSlab); [] switches the fan-out off, the multicast delta included.  At most 8 deltas,
        each a multiple of 16.  Only step() on the 8-envs-per-CTA kernel (Drift family, N <= 33 792) carries it: while it
        is set, rollout, act_step, the staged and host-transport steps and step() on another kernel variant raise WlError
        and leave the handle unchanged."""
        n = len(byte_deltas)
        arr = (C.c_int64 * max(1, n))(*byte_deltas)
        check(lib.wl_set_peer_fanout(self._h, n, arr), "wl_set_peer_fanout")

    def set_multicast_fanout(self, mc_byte_delta: int):
        """NVSwitch multicast alias of the symmetric buffer (SymmetricRolloutSlab.mc_delta): full output rows leave with one
        multimem.st replicated by the switch; 0 switches it off.  The other rows go peer by peer, so set_peer_fanout's
        deltas must be set first (WlError otherwise)."""
        check(lib.wl_set_multicast_fanout(self._h, int(mc_byte_delta)), "wl_set_multicast_fanout")

    def set_step_counter(self, value: int):
        check(lib.wl_set_step_counter(self._h, value, _stream_ptr(self.device)), "wl_set_step_counter")

    def advance_counter(self, k: int):
        """device counter base += k (a 1-thread kernel: capturable as the last node of a K-step graph)."""
        check(lib.wl_advance_counter(self._h, k, _stream_ptr(self.device)), "wl_advance_counter")

    def note_device_counter(self, value: int):
        """Tell the host mirror what the device counter base is after graph replays the library did not see."""
        check(lib.wl_note_device_counter(self._h, value), "wl_note_device_counter")

    def flush_log(self):
        """Publish the extras["log"] row of the most recent step now (otherwise the next step's launch does it).  Once this
        has run on the stream, that step's `log` tensor is no longer written and may be freed."""
        check(lib.wl_log_flush(self._h, _stream_ptr(self.device)), "wl_log_flush")

    @property
    def rew_weight(self) -> torch.Tensor:
        """Live reward weights (float32[8] view into the state buffer): what the next step will use / the last one used.
        The curriculum moves them between two slots on the device; the handle knows which one is current."""
        off = (int(lib.wl_reward_weights(self._h)) - self._buf.data_ptr()) // 4
        return self._buf[off: off + 8]

    def step(self, action: torch.Tensor, step_counter: int = -1, out=None, log: torch.Tensor | None = None):
        """action [N,2] f32 (device, contiguous) -> (obs [N,D] f32, rew [N] f32, terminated [N] u8, truncated [N] u8).
        `step_counter` = common_step_counter before the step, or device_counter_plus(k): the counter base kept on the device
        + k (CUDA-graph replayable: capture K steps k = 0..K-1, then advance_counter(K)).  Steps are issued with consecutive
        counters (a jump re-arms the episode log).  `log`: optional float32[16] device tensor receiving the episode-log row;
        it is written by the NEXT launch on this handle (the next step or flush_log())."""
        n = self.num_envs
        if out is None:
            obs = torch.empty((n, self.obs_dim), dtype=torch.float32, device=self.device)
            rew = torch.empty((n,), dtype=torch.float32, device=self.device)
            term = torch.empty((n,), dtype=torch.uint8, device=self.device)
            trunc = torch.empty((n,), dtype=torch.uint8, device=self.device)
        else:
            obs, rew, term, trunc = out
        check(lib.wl_step(self._h, C.c_void_p(action.data_ptr()), C.c_void_p(obs.data_ptr()), C.c_void_p(rew.data_ptr()),
                          C.c_void_p(term.data_ptr()), C.c_void_p(trunc.data_ptr()),
                          C.c_void_p(log.data_ptr()) if log is not None else None, step_counter,
                          _stream_ptr(self.device)), "wl_step")
        return obs, rew, term, trunc

    def make_host_io(self):
        """Buffers for step_host(): pinned host action / result blocks + their device twins."""
        n = self.num_envs
        nres = int(lib.wl_result_bytes(n))
        io = {
            "h_action": torch.empty((n, 2), dtype=torch.float32).pin_memory(),
            "d_action": torch.empty((n, 2), dtype=torch.float32, device=self.device),
            "d_result": torch.empty(nres, dtype=torch.uint8, device=self.device),
            "h_result": torch.empty(nres, dtype=torch.uint8).pin_memory(),
        }
        h = io["h_result"]
        io["rew"] = h[: 4 * n].view(torch.float32)
        io["terminated"] = h[4 * n: 5 * n].view(torch.bool)
        io["truncated"] = h[5 * n: 6 * n].view(torch.bool)
        d = io["d_result"]
        io["d_rew"] = d[: 4 * n].view(torch.float32)
        io["d_terminated"] = d[4 * n: 5 * n]
        io["d_truncated"] = d[5 * n: 6 * n]
        io["_p_h_action"] = C.c_void_p(io["h_action"].data_ptr())
        io["_p_h_result"] = C.c_void_p(io["h_result"].data_ptr())
        return io

    def step_host_zero_copy(self, io, step_counter: int, obs: torch.Tensor, log: torch.Tensor | None = None, p_obs=None, p_log=None,
                            p_action=None):
        """Zero-copy transport of the same contract: the kernel reads io.h_action / writes io.h_result over PCIe.
        p_obs / p_log: optional pre-built c_void_p of obs / log (saves two ctypes conversions per step); p_action: pointer
        of the CALLER's pinned [N,2] f32 action block, read in place instead of io.h_action."""
        if p_obs is None:
            p_obs = C.c_void_p(obs.data_ptr())
            p_log = C.c_void_p(log.data_ptr()) if log is not None else None
        rc = lib.wl_step_host_zero_copy(self._h, p_action if p_action is not None else io["_p_h_action"], p_obs, p_log,
                                        io["_p_h_result"], step_counter, _stream_ptr(self.device))
        if rc:
            check(rc, "wl_step_host_zero_copy")

    def step_host(self, io, step_counter: int, obs: torch.Tensor, log: torch.Tensor | None = None, h_obs: torch.Tensor | None = None,
                  p_action=None):
        """ONE C call: H2D(io.h_action) -> fused step -> D2H(reward | terminated | truncated) -> stream sync.
        Results are in io["rew"], io["terminated"], io["truncated"] (pinned host views); obs stays on the device."""
        check(lib.wl_step_host(self._h, p_action if p_action is not None else io["_p_h_action"], C.c_void_p(io["d_action"].data_ptr()),
                               C.c_void_p(obs.data_ptr()), C.c_void_p(io["d_result"].data_ptr()),
                               C.c_void_p(log.data_ptr()) if log is not None else None,
                               C.c_void_p(io["h_result"].data_ptr()),
                               C.c_void_p(h_obs.data_ptr()) if h_obs is not None else None, step_counter,
                               _stream_ptr(self.device)), "wl_step_host")

    def rollout(self, K: int, step_counter: int, slab, logs: torch.Tensor, actions: torch.Tensor | None = None):
        """K fused steps in ONE launch (wl_rollout): writes slab.obs/rewards/terminated/truncated[0:K] and logs[0:K];
        `actions` [K,N,2] or None (in-kernel U[-1,1]^2, stored to slab.actions).  With curriculum terms the window must end
        at or before the next episode boundary: use rollout_split() to cut a longer window."""
        check(lib.wl_rollout(self._h, K, C.c_void_p(actions.data_ptr()) if actions is not None else None,
                             C.c_void_p(slab.actions.data_ptr()) if actions is None else None,
                             C.c_void_p(slab.obs.data_ptr()), C.c_void_p(slab.rewards.data_ptr()),
                             C.c_void_p(slab.terminated.data_ptr()), C.c_void_p(slab.truncated.data_ptr()),
                             C.c_void_p(logs.data_ptr()), step_counter, _stream_ptr(self.device)), "wl_rollout")

    def camera(self, step_counter: int, obs: torch.Tensor, aug: torch.Tensor | None = None):
        """Visual task camera term alone (wl_camera): fills the first obs_dim - 8 floats of every row of `obs` [N, obs_dim].
        aug: None (drawn) or 9 floats on the device: brightness, contrast, saturation, hue, sigma, order[4]."""
        check(lib.wl_camera(self._h, C.c_void_p(obs.data_ptr()), step_counter, C.c_void_p(aug.data_ptr()) if aug is not None else None,
                            _stream_ptr(self.device)), "wl_camera")
        return obs

    def step_stage_a(self, action: torch.Tensor, step_counter: int, rew: torch.Tensor | None = None, term_bits: torch.Tensor | None = None):
        """Sections A-E of env.step (wl_step_stage_a): integrator + built-in terms; leaves the PRE-RESET state in the buffer.
        Returns (built-in reward [N] f32, termination bits [N] u8: bit j = built-in term j)."""
        n, dev = self.num_envs, self.device
        rew = rew if rew is not None else torch.empty(n, dtype=torch.float32, device=dev)
        term_bits = term_bits if term_bits is not None else torch.empty(n, dtype=torch.uint8, device=dev)
        check(lib.wl_step_stage_a(self._h, C.c_void_p(action.data_ptr()), C.c_void_p(rew.data_ptr()), C.c_void_p(term_bits.data_ptr()),
                                  step_counter, _stream_ptr(dev)), "wl_step_stage_a")
        return rew, term_bits

    def step_stage_b(self, term_bits: torch.Tensor, step_counter: int, extra_terminated: torch.Tensor | None = None,
                     extra_truncated: torch.Tensor | None = None, out=None, log: torch.Tensor | None = None):
        """Sections F-I (wl_step_stage_b): episode log, auto-reset of done envs (built-in bits | extras), commands /
        pushes, observations.  extras: [N] u8/bool or None.  Returns (obs, terminated u8, truncated u8)."""
        n, dev = self.num_envs, self.device
        if out is None:
            out = (torch.empty((n, self.obs_dim), dtype=torch.float32, device=dev), torch.empty(n, dtype=torch.uint8, device=dev),
                   torch.empty(n, dtype=torch.uint8, device=dev))
        obs, term, trunc = out
        u8 = lambda x: None if x is None else C.c_void_p((x.view(torch.uint8) if x.dtype == torch.bool else x).data_ptr())
        check(lib.wl_step_stage_b(self._h, C.c_void_p(term_bits.data_ptr()), u8(extra_terminated), u8(extra_truncated),
                                  C.c_void_p(obs.data_ptr()), C.c_void_p(term.data_ptr()), C.c_void_p(trunc.data_ptr()),
                                  C.c_void_p(log.data_ptr()) if log is not None else None, step_counter, _stream_ptr(dev)),
              "wl_step_stage_b")
        return obs, term, trunc

    def step_stage_b1(self, term_bits: torch.Tensor, step_counter: int, extra_terminated: torch.Tensor | None = None,
                      extra_truncated: torch.Tensor | None = None, out=None, log: torch.Tensor | None = None):
        """Sections F and H (wl_step_stage_b1): episode log, auto-reset of done envs (built-in bits | extras), the built-in
        interval pushes; the post-reset state is left in the buffer for host-side event terms.  Returns (terminated u8,
        truncated u8)."""
        n, dev = self.num_envs, self.device
        if out is None:
            out = (torch.empty(n, dtype=torch.uint8, device=dev), torch.empty(n, dtype=torch.uint8, device=dev))
        term, trunc = out
        u8 = lambda x: None if x is None else C.c_void_p((x.view(torch.uint8) if x.dtype == torch.bool else x).data_ptr())
        check(lib.wl_step_stage_b1(self._h, C.c_void_p(term_bits.data_ptr()), u8(extra_terminated), u8(extra_truncated),
                                   C.c_void_p(term.data_ptr()), C.c_void_p(trunc.data_ptr()),
                                   C.c_void_p(log.data_ptr()) if log is not None else None, step_counter, _stream_ptr(dev)),
              "wl_step_stage_b1")
        return term, trunc

    def step_stage_b2(self, step_counter: int, out: torch.Tensor | None = None) -> torch.Tensor:
        """Sections G and I (wl_step_stage_b2): commands and the observation of the state as it is now, at the counter the
        preceding step_stage_b1 was given."""
        obs = out if out is not None else torch.empty((self.num_envs, self.obs_dim), dtype=torch.float32, device=self.device)
        check(lib.wl_step_stage_b2(self._h, C.c_void_p(obs.data_ptr()), step_counter, _stream_ptr(self.device)), "wl_step_stage_b2")
        return obs

    def set_event_timers(self, ranges):
        """The interval timers of host-side interval event terms (wl_set_event_timers): a list of (lo, hi) interval_range_s,
        at most 8; each env's timers are drawn now.  [] frees them."""
        n = len(ranges)
        arr = (C.c_float * max(2, 2 * n))(*[float(v) for r in ranges for v in r])
        with torch.cuda.device(self.device):
            check(lib.wl_set_event_timers(self._h, n, arr), "wl_set_event_timers")

    def event_timers(self, done: torch.Tensor, step_counter: int, fired: torch.Tensor) -> torch.Tensor:
        """One step of the interval timers (wl_event_timers): redraw where `done` [N] (u8 / bool), count down, fire.
        Writes fired [n_terms, N] u8 (1: the term fires for the env in this step) and returns it."""
        d = done.view(torch.uint8) if done.dtype == torch.bool else done
        check(lib.wl_event_timers(self._h, C.c_void_p(d.data_ptr()), C.c_void_p(fired.data_ptr()), step_counter,
                                  _stream_ptr(self.device)), "wl_event_timers")
        return fired

    def set_device_terms(self, terms):
        """The handle's device terms (wl_set_device_terms): a list of (kind, role, weight, params[<= 4]) in evaluation
        order; [] clears them.  Resets their per-env state (episode sums, elevation_continuity's previous elevation)."""
        n = len(terms)
        arr = (_lib.WlTermDesc * max(1, n))()
        for k, (kind, role, weight, params) in enumerate(terms):
            p = list(params) + [0.0] * (4 - len(params))
            arr[k] = _lib.WlTermDesc(int(kind), int(role), float(weight), (C.c_double * 4)(*p))
        with torch.cuda.device(self.device):
            check(lib.wl_set_device_terms(self._h, arr, n), "wl_set_device_terms")

    @property
    def device_term_masks(self) -> torch.Tensor | None:
        """uint8 [N] view: bit k = device term k fired in the most recent step_terms (None without device terms)."""
        ptr = lib.wl_device_term_masks(self._h)
        if not ptr:
            return None
        if getattr(self, "_dt_masks", None) is None or self._dt_masks.data_ptr() != ptr:
            self._dt_masks = _device_u8_view(ptr, self.num_envs, self.device)
        return self._dt_masks

    def step_terms(self, action: torch.Tensor, step_counter: int = -1, out=None, log: torch.Tensor | None = None,
                   term_log: torch.Tensor | None = None):
        """step() with the device terms between stage a and stage b (wl_step_terms): same arguments and outputs, plus
        `term_log` (float32[8] device tensor or None) receiving the device terms' Episode_* entries of this step."""
        n = self.num_envs
        if out is None:
            out = (torch.empty((n, self.obs_dim), dtype=torch.float32, device=self.device), torch.empty(n, dtype=torch.float32, device=self.device),
                   torch.empty(n, dtype=torch.uint8, device=self.device), torch.empty(n, dtype=torch.uint8, device=self.device))
        obs, rew, term, trunc = out
        ptr = lambda x: C.c_void_p(x.data_ptr()) if x is not None else None
        check(lib.wl_step_terms(self._h, ptr(action), ptr(obs), ptr(rew), ptr(term), ptr(trunc), ptr(log), ptr(term_log),
                                step_counter, _stream_ptr(self.device)), "wl_step_terms")
        return obs, rew, term, trunc

    def set_device_events(self, terms):
        """The handle's device event terms (wl_set_device_events): a list of (mode, interval_range_s or None, velocity
        ranges [6] of (lo, hi) in x, y, z, roll, pitch, yaw order), applied in this order; the interval terms' timers are
        drawn now.  [] clears them.  From then on only step_terms steps the handle."""
        n = len(terms)
        arr = (_lib.WlDeviceEventDesc * max(1, n))()
        for k, (mode, interval_range_s, ranges) in enumerate(terms):
            d = arr[k]
            d.mode = _lib.WL_EVENT_MODE[mode]
            d.interval_range_s[0], d.interval_range_s[1] = interval_range_s if interval_range_s is not None else (0.0, 0.0)
            for j, (lo, hi) in enumerate(ranges):
                d.velocity_range[j][0], d.velocity_range[j][1] = float(lo), float(hi)
        with torch.cuda.device(self.device):
            check(lib.wl_set_device_events(self._h, arr, n), "wl_set_device_events")

    def device_events(self, terminated: torch.Tensor, truncated: torch.Tensor, step_counter: int):
        """The device event terms of one step on the state (wl_device_events), with the done bytes stage b1 wrote."""
        u8 = lambda x: C.c_void_p((x.view(torch.uint8) if x.dtype == torch.bool else x).data_ptr())
        check(lib.wl_device_events(self._h, u8(terminated), u8(truncated), step_counter, _stream_ptr(self.device)), "wl_device_events")

    def set_critic_terms(self, terms):
        """The handle's critic observation (wl_set_critic_terms): a list of term names of the library
        (``_lib.WL_CRITIC_TERMS``) or (name, clip) pairs, concatenated in this order into the critic row; [] clears it.
        Returns Dc, the row's width.  Nothing is launched; a graph captured earlier keeps the table it was captured with."""
        pairs = [(t, 0.0) if isinstance(t, str) else (t[0], t[1] or 0.0) for t in terms]
        for name, _ in pairs:
            if name not in _lib.WL_CRITIC_TERMS:
                raise ValueError(f"critic term {name!r} is not in the library {sorted(_lib.WL_CRITIC_TERMS)}")
        arr = (_lib.WlCriticTerm * max(1, len(pairs)))()
        for k, (name, clip) in enumerate(pairs):
            arr[k] = _lib.WlCriticTerm(_lib.WL_CRITIC_TERMS[name][0], float(clip))
        check(lib.wl_set_critic_terms(self._h, arr, len(pairs)), "wl_set_critic_terms")
        return self.critic_obs_dim

    def set_reset_events(self, material: bool = False, actuator_gains: bool = False, base_mass: bool = False,
                         wheel_mass: bool = False) -> int:
        """IsaacLab's mode="reset" for the start-up DR events (wl_set_reset_events): each event switched on here is drawn
        again, on the device, for every env a step auto-resets or reset() resets; the others keep their start-up values.  All
        False restores start-up DR.  Raises WlError, leaving the handle as it was, for an event the config does not have.
        Nothing is launched; a graph captured earlier keeps the events it was captured with.  Returns the mask."""
        on = {"material": material, "actuator_gains": actuator_gains, "base_mass": base_mass, "wheel_mass": wheel_mass}
        mask = sum(bit for name, bit in _lib.WL_RESET_EVENTS.items() if on[name])
        check(lib.wl_set_reset_events(self._h, mask), "wl_set_reset_events")
        return mask

    @property
    def reset_events(self) -> int:
        """The handle's WL_RESET_EV_* mask (0: every DR event in start-up mode)."""
        return int(lib.wl_reset_events(self._h))

    @property
    def critic_obs_dim(self) -> int:
        return int(lib.wl_critic_obs_dim(self._h))

    def critic_observe(self, out: torch.Tensor | None = None) -> torch.Tensor:
        """The critic row [N, Dc] of the current state (wl_critic_observe): after step(), the post-reset state its
        observation was formed from.  No noise, no counter; capturable."""
        dc = self.critic_obs_dim
        obs = out if out is not None else torch.empty((self.num_envs, dc), dtype=torch.float32, device=self.device)
        if dc and (obs.dtype != torch.float32 or tuple(obs.shape) != (self.num_envs, dc) or not obs.is_contiguous()
                   or not obs.is_cuda or obs.device.index != self.device.index):
            raise ValueError(f"out must be a contiguous float32 [{self.num_envs}, {dc}] tensor on {self.device} (the table's row "
                             f"is {dc} floats wide), not {obs.dtype} {tuple(obs.shape)} on {obs.device}")
        check(lib.wl_critic_observe(self._h, C.c_void_p(obs.data_ptr()), _stream_ptr(self.device)), "wl_critic_observe")
        return obs

    def set_policy_terms(self, terms) -> int:
        """The handle's policy observation table (wl_set_policy_terms): a list of ``(library name, noise, clip, scale)``
        (``policy_obs.lower_term``'s form; a bare name is a term without noise, clip or scale), concatenated in this order
        into the policy row; [] clears it.  Returns Dp.  Nothing is launched; a graph captured earlier keeps its table."""
        terms, arr = _policy_term_array(terms, _lib.WL_POLICY_TERMS, "policy term")
        check(lib.wl_set_policy_terms(self._h, arr, len(terms)), "wl_set_policy_terms")
        return self.policy_obs_dim

    def set_row_terms(self, terms) -> int:
        """The handle's row terms (wl_set_row_terms, DESIGN 6r): noise, clip and scale on the Elevation or Visual built-in
        row, one ``(name, noise, clip, scale)`` per term of the row in row order (``row_terms.lower_term``'s form; a bare
        name has none of them, so it is the raw value); [] clears them.  The names are the row's own
        (``_lib.WL_ROW_TASK_TERMS``).  Returns the number of terms.  Nothing is launched; a graph captured earlier keeps the
        terms it was captured with."""
        terms, arr = _policy_term_array(terms, _lib.WL_ROW_TERMS, "row term")
        check(lib.wl_set_row_terms(self._h, arr, len(terms)), "wl_set_row_terms")
        return self.row_terms

    def set_row_critic(self, row_terms, extra=()) -> int:
        """The handle's row critic (wl_set_row_critic, DESIGN 6s; Elevation only): the critic row is the Elevation row's six
        terms in row order, noise-free, each with its own clip and scale (``set_row_terms``'s form; a term with noise or a
        height map without a clip is refused), then the critic-library terms ``extra`` (``set_critic_terms``'s form).
        ``critic_observe`` writes it; [] clears it.  Returns Dc (689..721).  Nothing is launched; a graph captured earlier
        keeps the critic it was captured with."""
        row_terms, arr = _policy_term_array(row_terms, _lib.WL_ROW_TERMS, "row term")
        pairs = [(t, 0.0) if isinstance(t, str) else (t[0], t[1] or 0.0) for t in extra]
        for name, _ in pairs:
            if name not in _lib.WL_CRITIC_TERMS:
                raise ValueError(f"critic term {name!r} is not in the library {sorted(_lib.WL_CRITIC_TERMS)}")
        ex = (_lib.WlCriticTerm * max(1, len(pairs)))()
        for k, (name, clip) in enumerate(pairs):
            ex[k] = _lib.WlCriticTerm(_lib.WL_CRITIC_TERMS[name][0], float(clip))
        check(lib.wl_set_row_critic(self._h, arr, len(row_terms), ex, len(pairs)), "wl_set_row_critic")
        return self.critic_obs_dim

    @property
    def row_terms(self) -> int:
        """The number of row terms of the handle (0: the built-in row)."""
        return int(lib.wl_row_terms(self._h))

    @property
    def policy_obs_dim(self) -> int:
        """Dp, the width of the policy row of the handle's table (0 without one; sim.obs_dim stays the built-in width)."""
        return int(lib.wl_policy_obs_dim(self._h))

    @property
    def policy_width(self) -> int:
        """The width of the row the policy reads: Dp with a policy table, else obs_dim (the policy kernels read the same)."""
        return self.policy_obs_dim or self.obs_dim

    def observe_policy_row(self, step_counter: int, call_idx: int, out: torch.Tensor) -> torch.Tensor:
        """observation_manager.compute()'s policy row into `out` [N, policy_width]: wl_observe, or with a policy table
        wl_policy_observe at the same call index."""
        if self.policy_obs_dim:
            return self.policy_observe(step_counter, call_idx, out=out)
        return self.observe(step_counter, call_idx, out=out)

    def policy_observe(self, step_counter: int, call_idx: int | None = None, out: torch.Tensor | None = None) -> torch.Tensor:
        """The policy row [N, Dp] of the table (wl_policy_observe) from the current state: with call_idx None the row of the
        step just taken at `step_counter` (a host value or WL_DEVICE_COUNTER_PLUS(k)), else the row of
        observe(step_counter, call_idx).  Capturable."""
        dp = self.policy_obs_dim
        obs = out if out is not None else torch.empty((self.num_envs, dp), dtype=torch.float32, device=self.device)
        if dp and (obs.dtype != torch.float32 or tuple(obs.shape) != (self.num_envs, dp) or not obs.is_contiguous()
                   or not obs.is_cuda or obs.device.index != self.device.index):
            raise ValueError(f"out must be a contiguous float32 [{self.num_envs}, {dp}] tensor on {self.device} (the table's row "
                             f"is {dp} floats wide), not {obs.dtype} {tuple(obs.shape)} on {obs.device}")
        ci = _lib.WL_POLICY_OBS_AFTER_STEP if call_idx is None else int(call_idx)
        check(lib.wl_policy_observe(self._h, step_counter, ci, C.c_void_p(obs.data_ptr()), _stream_ptr(self.device)), "wl_policy_observe")
        return obs

    def observe(self, step_counter: int, call_idx: int = 0, out: torch.Tensor | None = None):
        obs = out if out is not None else torch.empty((self.num_envs, self.obs_dim), dtype=torch.float32, device=self.device)
        check(lib.wl_observe(self._h, C.c_void_p(obs.data_ptr()), step_counter, call_idx, _stream_ptr(self.device)),
              "wl_observe")
        return obs

    def bind_step(self, action: torch.Tensor, out, log: torch.Tensor | None = None):
        """Pre-resolve the pointers of one (action, outputs) set; returns f(step_counter) that enqueues the step with a
        single ctypes call (used by tight host loops that reuse the same buffers, e.g. rollout slabs)."""
        obs, rew, term, trunc = out
        args = (self._h, C.c_void_p(action.data_ptr()), C.c_void_p(obs.data_ptr()), C.c_void_p(rew.data_ptr()),
                C.c_void_p(term.data_ptr()), C.c_void_p(trunc.data_ptr()), C.c_void_p(log.data_ptr()) if log is not None else None)
        keep = (action, obs, rew, term, trunc, log)
        fn, dev = lib.wl_step, self.device

        def run(step_counter: int, _keep=keep):
            rc = fn(*args, step_counter, _stream_ptr(dev))
            if rc:
                check(rc, "wl_step")
        return run

    def curriculum(self, slots, increases, fire_mask: int):
        n = len(slots)
        if n == 0 or fire_mask == 0:
            return
        a = (C.c_int32 * n)(*slots)
        b = (C.c_float * n)(*increases)
        check(lib.wl_curriculum(self._h, n, a, b, fire_mask, _stream_ptr(self.device)), "wl_curriculum")

    def synth_actions(self, step_counter: int, dist: int = 0, out: torch.Tensor | None = None):
        act = out if out is not None else torch.empty((self.num_envs, 2), dtype=torch.float32, device=self.device)
        check(lib.wl_synth_actions(self._h, C.c_void_p(act.data_ptr()), step_counter, dist, _stream_ptr(self.device)),
              "wl_synth_actions")
        return act

    def suspension_state(self):
        """Derived suspension joint (pos [N,4], vel [N,4]) in wheel order [bl, br, fl, fr]."""
        pos = torch.empty((self.num_envs, 4), dtype=torch.float32, device=self.device)
        vel = torch.empty((self.num_envs, 4), dtype=torch.float32, device=self.device)
        check(lib.wl_derive_suspension(self._h, C.c_void_p(pos.data_ptr()), C.c_void_p(vel.data_ptr()), _stream_ptr(self.device)),
              "wl_derive_suspension")
        return pos, vel

    def set_scan_tma(self, mode):
        """Height-scan tile staging: 1/True one TMA tile per CTA (default), 2 TMA producer/consumer pipeline, 0/False plain loads."""
        check(lib.wl_set_scan_tma(self._h, int(mode)), "wl_set_scan_tma")

    def set_kernel_variant(self, lanes_per_env: int):
        """0 auto, 1 thread-per-env, 4 quad-per-env, 8 quad + aux warp (Drift family); bit-identical results."""
        check(lib.wl_set_kernel_variant(self._h, lanes_per_env), "wl_set_kernel_variant")

    @property
    def launch_count(self) -> int:
        return int(lib.wl_launch_count(self._h))

    @property
    def chained_step_count(self) -> int:
        """wl_step launches of the duo kernel that ran chained after another env set's step (DESIGN.md 6e)."""
        return int(lib.wl_chained_step_count(self._h))

    @property
    def deep_step_count(self) -> int:
        """Of the chained steps, the ones that ran deep: triggered the next launch at entry (DESIGN.md 6e)."""
        return int(lib.wl_deep_step_count(self._h))

    # -- zero-copy state views (IsaacLab ArticulationData names) -------------------------------------
    @property
    def root_pos_w(self):
        return self.groups[G_POS, :, 0:3]

    @property
    def root_quat_w(self):
        return self.groups[G_QUAT]

    @property
    def root_lin_vel_w(self):
        return self.groups[G_LINVEL, :, 0:3]

    @property
    def root_ang_vel_w(self):
        return self.groups[G_ANGVEL, :, 0:3]

    @property
    def wheel_vel(self):
        return self.groups[G_WHEEL]

    @property
    def steer_pos(self):
        return self.groups[G_STEER, :, 0:2]

    @property
    def steer_vel(self):
        return self.groups[G_STEER, :, 2:4]

    @property
    def episode_length_buf(self):
        return self.groups[G_POS, :, 3].view(torch.int32)

    @property
    def last_action(self):
        return self.groups[G_ACTION, :, 0:2]

    @property
    def prev_action(self):
        return self.groups[G_ACTION, :, 2:4]

    @property
    def episode_sums(self):
        return torch.cat([self.groups[G_SUM0], self.groups[G_SUM1]], dim=-1)

    def state_snapshot(self) -> torch.Tensor:
        """Copy of the whole state buffer (groups + globals) for checkpoint / parity tests."""
        return self._buf.clone()

    def load_state(self, buf: torch.Tensor):
        self._buf.copy_(buf.to(self.device))
