"""The Drift step kernel's peer fan-out (wl_set_peer_fanout, wl_step_duo_kernel<1, 0>) on one GPU, against the CPU oracle.

The kernel stores every output row locally and at pointer + delta for each peer delta, through plain generic addresses, so
a "peer" can be another buffer on the same device.  That runs the general fan-out form bit for bit on one H100:
- ranks emulated on one device, laid out as SymmetricRolloutSlab lays them out, for 2, 3 and 9 ranks (8 peers);
- same-device mirrors of one handle's outputs: the packed path (full CTA, 16-byte aligned rows) and the element-wise path
  (ragged last CTA, rows at 8-, 4-, 1- and 3-byte offsets), with positive and negative deltas;
- the shipped and lowered Drift-family cfgs on the fan-out instantiation, and the hand-back to the spec instantiation;
- fan-out switched on, off and between mirror sets from step to step, eagerly and in one CUDA graph, across t = 250;
- the calls that must refuse while a fan-out is set, and that a refused call leaves the handle as it was.

Every output is compared bit for bit, the episode-log sums to rtol 1e-5.  Every buffer is filled with the 0xA5 sentinel
first, and every byte the fan-out does not own must still hold it afterwards.  Every pointer + delta this file hands the
library is memory the test owns, even for calls that ought to be refused; no step is launched while a multicast delta or
a delta that is not a multiple of 16 is set."""
import ctypes as C

import numpy as np
import pytest

import oracle_lib as O
from test_duo_coverage_gpu import SPECIALISED, WIDE, _bits, _check_log, _check_step, _launch_info, _need_gpu, _spec, _synth, _wide_actions

torch = pytest.importorskip("torch")

SENT = 0xA5
DEV = "cuda:0"
OBS_BYTES = 14 * 4                                          # one Drift observation row


def _align(x, a):
    return (x + a - 1) // a * a


def _sentinel(nbytes):
    return torch.full((nbytes,), SENT, dtype=torch.uint8, device=DEV)


def _wl():
    import wheeledlab_b200 as wl
    return wl


# ---- same-device mirrors ---------------------------------------------------------------------------------------------
class _Arena:
    """One sentinel-filled device buffer holding `n_slots` copies of an output region, `D` bytes apart (a multiple of 16,
    not of 256).  A region holds T rows of obs [n, 14] f32, reward [n] f32, terminated [n] u8 and truncated [n] u8, each
    block placed `offsets` bytes past a 16-byte boundary and at least 64 sentinel bytes after the block before it.  The
    handle writes slot `primary`; the other slots are its mirrors, at deltas (slot - primary) * D."""

    def __init__(self, n, T, n_slots, primary, offsets=(0, 0, 0, 0)):
        self.n, self.T, self.n_slots, self.primary = n, T, n_slots, primary
        self.rows = (n * OBS_BYTES, n * 4, n, n)            # bytes of one step's row of each block
        self.fields, off = [], 0
        for row, o in zip(self.rows, offsets):
            off = _align(off + 64, 16) + o
            self.fields.append(off)
            off += row * T
        self.S = _align(off + 64, 16)
        self.D = _align(self.S, 256) + 48
        self.buf = _sentinel(256 + n_slots * self.D + 256)
        owned = np.zeros(self.buf.numel(), bool)
        for s in range(n_slots):
            for f, row in zip(self.fields, self.rows):
                owned[self.slot(s) + f: self.slot(s) + f + row * T] = True
        self.owned = owned

    def slot(self, s):
        return 256 + s * self.D

    def delta(self, s):
        return (s - self.primary) * self.D

    def outputs(self, t):
        """Row t of the primary slot as the (obs, rew, terminated, truncated) tensors wl_step writes."""
        b, n = self.slot(self.primary), self.n
        v = [self.buf[b + f + t * row: b + f + (t + 1) * row] for f, row in zip(self.fields, self.rows)]
        return v[0].view(torch.float32).view(n, 14), v[1].view(torch.float32), v[2], v[3]

    def host_rows(self, a, s, t):
        """Row t of slot s of the host copy `a`, as four byte arrays."""
        b = self.slot(s)
        return [a[b + f + t * row: b + f + (t + 1) * row] for f, row in zip(self.fields, self.rows)]

    def host_outputs(self, a, t):
        o, r, te, tr = (x.copy() for x in self.host_rows(a, self.primary, t))
        return o.view(np.float32).reshape(self.n, 14), r.view(np.float32), te, tr

    def check_bytes(self, a, attached, what):
        """Mirror slot s holds the primary's rows of the steps in attached[s] (a set of row indices) and the sentinel
        everywhere else; nothing outside the blocks changed in any slot."""
        assert (a[~self.owned] == SENT).all(), f"{what}: a byte outside the output blocks changed"
        for s in range(self.n_slots):
            if s == self.primary:
                continue
            for t in range(self.T):
                got, ref = self.host_rows(a, s, t), self.host_rows(a, self.primary, t)
                for g, r in zip(got, ref):
                    if t in attached.get(s, ()):
                        assert np.array_equal(g, r), f"{what}: mirror slot {s} row {t} differs from the primary"
                    else:
                        assert (g == SENT).all(), f"{what}: mirror slot {s} row {t} written while not attached"


LAYOUTS = {"aligned": (0, 0, 0, 0), "offset": (8, 4, 1, 3)}  # offset: obs 8- but not 16-byte aligned, reward +4, masks +1 / +3


def _mirrored_run(spec, n_mirrors, layout, steps, action_fn=_synth, term_bits=False):
    """One handle stepping `steps` times with `n_mirrors` same-device mirrors attached; every step against the oracle, every
    mirror byte-identical to the primary, no other byte changed.  Returns (sim, orc, threads per CTA of the fan-out run)."""
    wl = _wl()
    n = int(spec.cfg.num_envs)
    ar = _Arena(n, 1, n_mirrors + 1, n_mirrors // 2, LAYOUTS[layout])
    mirrors = [s for s in range(ar.n_slots) if s != ar.primary]
    deltas = [ar.delta(s) for s in mirrors]
    assert all(d % 16 == 0 and d % 256 != 0 for d in deltas) and (n_mirrors == 1 or min(deltas) < 0 < max(deltas))
    sim = wl.WheeledSim(spec, DEV); sim.startup(); sim.reset(None, 0)
    orc = O.Oracle(spec.cfg, threads=8); orc.startup(); orc.reset(None, 0)
    bits = torch.full((n,), SENT, dtype=torch.uint8, device=DEV) if term_bits else None
    if bits is not None:
        wl._lib.check(wl.lib.wl_set_term_bits(sim._h, C.c_void_p(bits.data_ptr())), "wl_set_term_bits")
    w0 = sim.rew_weight.cpu().numpy().copy()
    sim.set_peer_fanout(deltas)
    n_done, threads = 0, None
    for t in range(steps):
        act = action_fn(sim, t)
        log = torch.empty(16, device=DEV)
        sim.step(act, t, out=ar.outputs(0), log=log)
        sim.flush_log()
        variant, _, specialised, th = _launch_info(sim)
        assert (variant, specialised) == (8, 0), (variant, specialised)
        assert threads in (None, th) and th in (64, 96), th
        threads = th
        a = ar.buf.cpu().numpy()
        ref = orc.step(act.cpu().numpy(), t)
        n_done += _check_step(ar.host_outputs(a, 0), ref, f"step {t}")
        _check_log(log.cpu().numpy(), orc.log(), f"step {t}")
        ar.check_bytes(a, {s: {0} for s in mirrors}, f"step {t}")
        if bits is not None:
            want = ref[3] | (ref[2] << 1)                    # Drift term order: bit 0 time_out, bit 1 out_of_bounds
            assert np.array_equal(bits.cpu().numpy(), want), f"step {t}: termination-term bits differ"
    if bits is not None:
        wl._lib.check(wl.lib.wl_set_term_bits(sim._h, None), "wl_set_term_bits")
    assert np.array_equal(_bits(sim.groups.cpu().numpy()), _bits(orc.export_state())), "final state differs"
    assert np.array_equal(_bits(sim.rew_weight.cpu().numpy()), _bits(orc.weights())), "reward weights differ"
    if spec.cfg.term_enable:
        assert n_done > 0, "trajectory too short to exercise the auto-reset"
    if spec.cfg.curr_n > 0 and steps > spec.cfg.max_episode_length:
        assert not np.array_equal(sim.rew_weight.cpu().numpy(), w0), "the curriculum boundary did not move the weights"
    return sim, orc, threads


# ---- 1. ranks emulated on one device ---------------------------------------------------------------------------------
EMU_T = 260                                                 # crosses the episode / curriculum boundary at t = 250


@pytest.mark.gpu
@pytest.mark.parametrize("n_local", [8, 333, 2048])
@pytest.mark.parametrize("world", [2, 3, 9])
def test_emulated_ranks_gather_the_rollout(world, n_local):
    """`world` handles on one device, rank r with env_id_offset r * n_local, each with one flat buffer of world x slab bytes
    whose slot r is its RolloutSlab and peer deltas computed as SymmetricRolloutSlab computes them (9 ranks: 8 peers).
    Afterwards every buffer holds every rank's obs / reward / done rows, nothing else of a peer's slot was written, each
    rank matches its own oracle (outputs and log), and the gathered rollout equals one world x n_local handle without
    fan-out, itself checked against the oracle."""
    _need_gpu()
    wl = _wl()
    from wheeledlab_b200.distributed import GatheredRollout, RolloutSlab, slab_nbytes
    T, N, W = EMU_T, n_local, world
    nb = slab_nbytes(T, N, 14, 2)
    bufs = [_sentinel(W * nb) for _ in range(W)]
    slabs = [RolloutSlab(T, N, 14, 2, DEV, flat=bufs[r][r * nb:(r + 1) * nb]) for r in range(W)]
    sims, specs = [], []
    for r in range(W):
        spec = _spec("drift", N, seed=13)
        spec.cfg.env_id_offset = r * N
        s = wl.WheeledSim(spec, DEV); s.startup(); s.reset(None, 0)
        ptrs = [b.data_ptr() for b in bufs]
        s.set_peer_fanout([ptrs[p] - ptrs[r] for p in range(W) if p != r])
        sims.append(s); specs.append(spec)
    whole_spec = _spec("drift", W * N, seed=13)
    whole = wl.WheeledSim(whole_spec, DEV); whole.startup(); whole.reset(None, 0)
    whole_slab = RolloutSlab(T, W * N, 14, 2, DEV)
    logs = [torch.zeros((T, 16), device=DEV) for _ in range(W + 1)]
    acts = []
    for t in range(T):
        act = whole.synth_actions(t, dist=t % 2)
        acts.append(act)
        whole.step(act, t, out=whole_slab.step_outputs(t), log=logs[W][t])
        for r in range(W):
            slabs[r].actions[t].copy_(act[r * N:(r + 1) * N])   # what the caller records locally (the fan-out does not)
            sims[r].step(act[r * N:(r + 1) * N].contiguous(), t, out=slabs[r].step_outputs(t), log=logs[r][t])
            assert _launch_info(sims[r])[:3:2] == (8, 0)
    for s in sims + [whole]:
        s.flush_log()
    torch.cuda.synchronize()
    # bytes: slot p of every buffer holds exactly rank p's fanned fields; the rest of every peer slot is sentinel
    p0 = slabs[0]
    own = torch.zeros(nb, dtype=torch.bool, device=DEV)
    off = 0
    for k, size in p0._sizes.items():
        if k == "obs":
            own[off + N * OBS_BYTES: off + size] = True         # rows 1..T; obs_in[0] is the caller's
        elif k != "actions":
            own[off: off + size] = True
        off += _align(size, 256)
    for r in range(W):
        view = bufs[r].view(W, nb)
        for p in range(W):
            if p != r:
                assert torch.equal(view[p][own], slabs[p].flat[own]), f"buffer {r}: slot {p} differs from rank {p}'s rows"
                assert bool((view[p][~own] == SENT).all()), f"buffer {r}: a byte of slot {p} the fan-out does not own changed"
            else:
                assert bool((view[p][~own & ~_actions_mask(p0, nb)] == SENT).all()), f"buffer {r}: padding or obs_in[0] written"
    # the oracle, rank by rank and for the whole handle
    orcs = [O.Oracle(sp.cfg, threads=8) for sp in specs]
    ow = O.Oracle(whole_spec.cfg, threads=8)
    for o in orcs + [ow]:
        o.startup(); o.reset(None, 0)
    host = [{k: getattr(sl, k).cpu().numpy() for k in ("obs", "rewards", "terminated", "truncated")} for sl in slabs + [whole_slab]]
    hlogs = [lg.cpu().numpy() for lg in logs]
    all_reset_at_boundary = True
    for t in range(T):
        a = acts[t].cpu().numpy()
        _check_step(tuple(host[W][k][t] for k in ("obs", "rewards", "terminated", "truncated")), ow.step(a, t), f"whole, step {t}")
        _check_log(hlogs[W][t], ow.log(), f"whole, step {t}")
        for r in range(W):
            ref = orcs[r].step(a[r * N:(r + 1) * N], t)
            _check_step(tuple(host[r][k][t] for k in ("obs", "rewards", "terminated", "truncated")), ref, f"rank {r}, step {t}")
            _check_log(hlogs[r][t], orcs[r].log(), f"rank {r}, step {t}")
            if t == 249:
                all_reset_at_boundary &= orcs[r].any_reset()
    # A rank whose envs all reset before t = 249 has none left to reset at the boundary, so (as with the reference's one
    # process per GPU) it does not advance its curriculum there and its rewards leave the single run's from then on.
    rows = T if all_reset_at_boundary else 250
    assert all_reset_at_boundary or N < 64, "every shard of >= 64 envs resets at the curriculum boundary"
    for r in range(W):
        g = GatheredRollout(bufs[r].view(W, nb), slabs[r])
        for k in ("obs", "rewards", "terminated", "truncated"):
            got, ref = g.cat(k)[:rows], getattr(whole_slab, k)[:rows]
            if got.dtype == torch.float32:
                got, ref = got.view(torch.int32), ref.view(torch.int32)
            assert torch.equal(got, ref), f"buffer {r}: gathered {k} differs from the {W * N}-env run"


def _actions_mask(slab, nb):
    m = torch.zeros(nb, dtype=torch.bool, device=DEV)
    off = 0
    for k, size in slab._sizes.items():
        if k == "actions":
            m[off: off + size] = True
        off += _align(size, 256)
    return m


# ---- 2. row paths and geometry ---------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("layout", list(LAYOUTS))
@pytest.mark.parametrize("n_mirrors", [1, 3, 8])
@pytest.mark.parametrize("n", [1, 7, 9, 333, 4096, 8197, 32 * 132 * 4 * 2])
def test_mirrors_of_every_row_path_match_oracle(n, n_mirrors, layout):
    """Packed rows (full CTA, 16-byte aligned) and element-wise rows (ragged last CTA; obs at +8 B, reward at +4 B, the
    masks at +1 / +3 B) fanned to 1, 3 and 8 same-device mirrors, 25-step episodes so every CTA resets within the run."""
    _need_gpu()
    spec = _spec("drift", n, seed=3)
    spec.cfg.max_episode_length = 25
    _, _, threads = _mirrored_run(spec, n_mirrors, layout, 30 if n < 30000 else 27)
    print(f"fan-out kernel at {n} envs: {threads} threads per CTA")


# ---- 3. configs on the fan-out instantiation -------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name,deviation", [(s, None) for s in SPECIALISED] + [("drift", "all")])
def test_configs_on_the_fanout_kernel_match_oracle(name, deviation):
    """The shipped and lowered Drift-family cfgs (and every step-spec field moved at once) run the fan-out kernel's generic
    body (specialised 0) with 3 mirrors; after set_peer_fanout([]) the next step runs the spec instantiation again.  The
    `drift` case also takes the per-env termination-term bits."""
    _need_gpu()
    n, steps = 333, 120
    spec = _spec(name, n, deviation=deviation)
    sim, orc, threads = _mirrored_run(spec, 3, "aligned", steps, _wide_actions if deviation in WIDE else _synth,
                                      term_bits=(name == "drift" and deviation is None))
    print(f"{name}/{deviation}: fan-out kernel at {n} envs: {threads} threads per CTA")
    sim.set_peer_fanout([])
    act = _synth(sim, steps)
    out = sim.step(act, steps)
    _check_step(out, orc.step(act.cpu().numpy(), steps), "first step without fan-out")
    variant, _, specialised, _ = _launch_info(sim)
    assert (variant, specialised) == (8, 1 if deviation is None else 0), (variant, specialised)


# ---- 4. toggling and graphs ------------------------------------------------------------------------------------------
TOGGLE_T = 262
SET_A, SET_B = [0], [1, 3, 4]                               # mirror slots around primary slot 2 (deltas -2D; -D, +D, +2D)
SCHEDULE = [None, SET_A, SET_B, SET_A, SET_B, None, SET_B]  # which mirror set step t has attached: SCHEDULE[t % 7]


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["eager", "graph"])
@pytest.mark.parametrize("n", [333, 4096])
def test_fanout_toggled_between_steps_matches_oracle(n, mode):
    """As bench.py's make_bound does: set_peer_fanout before each step, off / one mirror / three mirrors, eagerly and in one
    CUDA graph on the device counter, across t = 250.  Step t writes row t of a T-row region, so each mirror must hold
    exactly the rows of the steps it was attached for."""
    _need_gpu()
    wl = _wl()
    ar = _Arena(n, TOGGLE_T, 5, 2)
    spec = _spec("drift", n, seed=31)
    sim = wl.WheeledSim(spec, DEV); sim.startup(); sim.reset(None, 0)
    acts = torch.stack([sim.synth_actions(t, dist=t % 2) for t in range(TOGGLE_T)])
    logs = torch.zeros((TOGGLE_T, 16), device=DEV)
    w0 = sim.rew_weight.cpu().numpy().copy()
    graph = mode == "graph"

    def body():
        for t in range(TOGGLE_T):
            fan = SCHEDULE[t % 7]
            sim.set_peer_fanout([ar.delta(s) for s in fan] if fan else [])
            sim.step(acts[t], wl.WheeledSim.device_counter_plus(t) if graph else t, out=ar.outputs(t), log=logs[t])
        sim.set_peer_fanout([])
        if graph:
            sim.advance_counter(TOGGLE_T)

    sim.set_step_counter(0)
    if graph:
        g, s = torch.cuda.CUDAGraph(), torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            with torch.cuda.graph(g, stream=s):
                body()
        torch.cuda.current_stream().wait_stream(s)
        assert (ar.buf == SENT).all(), "capture ran a step"
        sim.set_step_counter(0)                               # (capture moved the host mirror only)
        g.replay()
    else:
        body()
    sim.flush_log()
    torch.cuda.synchronize()
    a = ar.buf.cpu().numpy()
    attached = {s: {t for t in range(TOGGLE_T) if SCHEDULE[t % 7] and s in SCHEDULE[t % 7]} for s in SET_A + SET_B}
    ar.check_bytes(a, attached, mode)
    orc = O.Oracle(spec.cfg, threads=8); orc.startup(); orc.reset(None, 0)
    hlogs, hacts = logs.cpu().numpy(), acts.cpu().numpy()
    for t in range(TOGGLE_T):
        _check_step(ar.host_outputs(a, t), orc.step(hacts[t], t), f"{mode} step {t}")
        _check_log(hlogs[t], orc.log(), f"{mode} step {t}")
    assert np.array_equal(_bits(sim.groups.cpu().numpy()), _bits(orc.export_state())), "final state differs"
    w = sim.rew_weight.cpu().numpy()
    assert np.array_equal(_bits(w), _bits(orc.weights())), "reward weights differ"
    assert not np.array_equal(w, w0), "the curriculum boundary did not move the weights"


# ---- 5. refusals, and no side effects --------------------------------------------------------------------------------
def _handle(n=333, seed=5):
    wl = _wl()
    spec = _spec("drift", n, seed=seed)
    sim = wl.WheeledSim(spec, DEV); sim.startup(); sim.reset(None, 0)
    orc = O.Oracle(spec.cfg, threads=8); orc.startup(); orc.reset(None, 0)
    return sim, orc


def _checked_step(sim, orc, t, log=None):
    """One step without fan-out against the oracle; returns the oracle's log row of the step."""
    act = _synth(sim, t)
    out = sim.step(act, t, log=log)
    _check_step(out, orc.step(act.cpu().numpy(), t), f"step {t}")
    return orc.log()


def _nan_log():
    """A log buffer that no published row matches by accident."""
    return torch.full((16,), float("nan"), device=DEV)


def _owned_delta(nbytes):
    """A delta that keeps pointer + delta inside a buffer of _owned_delta(n) + n bytes starting at the pointer."""
    return _align(nbytes, 256) + 16


def _prepare_call(kind, sim, t, fan_delta):
    """(buffers, call): `call` issues `kind` at step counter t into `buffers`, each sentinel-filled.  The host-transport steps
    pass their own result blocks to wl_step, so those, and the obs buffer, get `fan_delta` bytes of slack after them."""
    from wheeledlab_b200.distributed import RolloutSlab
    from wheeledlab_b200.policy import act_infer_step, act_step, pack_actor_critic
    n = sim.num_envs
    f32 = lambda *s: _sentinel(int(np.prod(s)) * 4).view(torch.float32).view(*s)
    out = (f32(n, 14), f32(n), _sentinel(n), _sentinel(n))
    act = _synth(sim, t)
    if kind in ("act_step", "act_infer_step"):
        torch.manual_seed(0)
        mk = lambda o: torch.nn.Sequential(torch.nn.Linear(14, 64), torch.nn.ELU(), torch.nn.Linear(64, 64), torch.nn.ELU(),
                                           torch.nn.Linear(64, o)).to(DEV)
        blob = pack_actor_critic(mk(2), mk(1), torch.tensor([0.7, 1.3], device=DEV), 14, DEV)
        obs_in = torch.zeros((n, 14), device=DEV)
        pol = (f32(n, 2), f32(n, 2), f32(n), f32(n))
        if kind == "act_step":
            return list(out) + list(pol), lambda: act_step(sim, obs_in, blob, *pol, out, None, t)
        return list(out) + [pol[0]], lambda: act_infer_step(sim, obs_in, blob, pol[0], out, None, t)
    if kind == "rollout":
        slab = RolloutSlab(2, n, 14, 2, DEV, flat=_sentinel(RolloutSlab(2, n, 14, 2, DEV).nbytes))
        lg = f32(2, 16)
        return [slab.flat, lg], lambda: sim.rollout(2, t, slab, lg)
    if kind == "stage_a":
        rew, bits = f32(n), _sentinel(n)
        return [rew, bits], lambda: sim.step_stage_a(act, t, rew=rew, term_bits=bits)
    if kind == "stage_b":
        bits = torch.zeros(n, dtype=torch.uint8, device=DEV)
        return [out[0], out[2], out[3]], lambda: sim.step_stage_b(bits, t, out=(out[0], out[2], out[3]))
    wl = _wl()
    nres = int(wl.lib.wl_result_bytes(n))
    obs_arena, res_arena = _sentinel(fan_delta + n * OBS_BYTES), _sentinel(fan_delta + nres)
    h_res = torch.full((fan_delta + nres,), SENT, dtype=torch.uint8).pin_memory()
    h_act = act.cpu().pin_memory()
    io = {"h_action": h_act, "d_action": torch.empty((n, 2), device=DEV), "d_result": res_arena, "h_result": h_res,
          "_p_h_action": C.c_void_p(h_act.data_ptr()), "_p_h_result": C.c_void_p(h_res.data_ptr())}
    obs = obs_arena[: n * OBS_BYTES].view(torch.float32).view(n, 14)
    fn = sim.step_host if kind == "step_host" else sim.step_host_zero_copy
    return [obs_arena, res_arena, h_res], lambda: fn(io, t, obs)


def _untouched(bufs, what):
    torch.cuda.synchronize()
    for k, b in enumerate(bufs):
        assert bool((b.reshape(-1).view(torch.uint8) == SENT).all()), f"{what}: buffer {k} of the refused call was written"


def _continues_like_the_oracle(sim, orc, t0, logs, ref_logs, t_end):
    """Steps t0..t_end-1 without fan-out against the oracle; then every log row and the state."""
    for t in range(t0, t_end):
        ref_logs[t] = _checked_step(sim, orc, t, logs[t])
    sim.flush_log()
    torch.cuda.synchronize()
    for t in range(t_end):
        _check_log(logs[t].cpu().numpy(), ref_logs[t], f"log of step {t}")
    assert np.array_equal(_bits(sim.groups.cpu().numpy()), _bits(orc.export_state())), "state differs"


FIX_LIST = ["rollout", "act_step", "act_infer_step", "stage_a", "stage_b", "step_host", "step_host_zero_copy"]


@pytest.mark.gpu
@pytest.mark.parametrize("kind", FIX_LIST)
def test_calls_that_cannot_fan_out_refuse_and_change_nothing(kind):
    """While a fan-out is set, every call that writes a step's rows without carrying it raises, writes nothing, and leaves
    the handle so that, with the fan-out cleared, it continues from the same counter, state and log as the oracle."""
    _need_gpu()
    from wheeledlab_b200._lib import WlError
    sim, orc = _handle()
    logs, ref = [_nan_log() for _ in range(5)], {}
    for t in range(2):
        ref[t] = _checked_step(sim, orc, t, logs[t])
    delta = _owned_delta(sim.num_envs * OBS_BYTES)
    bufs, call = _prepare_call(kind, sim, 2, delta)
    sim.set_peer_fanout([delta])
    with pytest.raises(WlError):
        call()
    _untouched(bufs, kind)
    sim.set_peer_fanout([])
    _continues_like_the_oracle(sim, orc, 2, logs, ref, 5)


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["variant1", "variant4", "n33793"])
def test_step_on_a_kernel_without_fanout_refuses_and_changes_nothing(case):
    """wl_step with a fan-out set on the thread-per-env and quad kernels (chosen with set_kernel_variant, or N = 33 793: the
    first size past the duo kernel) raises, and the handle is as it was."""
    _need_gpu()
    from wheeledlab_b200._lib import WlError
    sim, orc = _handle(n=32 * 132 * 4 * 2 + 1 if case == "n33793" else 333)
    n = sim.num_envs
    logs, ref = [_nan_log() for _ in range(5)], {}
    for t in range(2):
        ref[t] = _checked_step(sim, orc, t, logs[t])
    ar = _Arena(n, 1, 2, 0)
    if case != "n33793":
        sim.set_kernel_variant(1 if case == "variant1" else 4)
    sim.set_peer_fanout([ar.delta(1)])
    with pytest.raises(WlError, match="variant 8"):
        sim.step(_synth(sim, 2), 2, out=ar.outputs(0), log=logs[2])
    _untouched([ar.buf], case)
    sim.set_peer_fanout([])
    _continues_like_the_oracle(sim, orc, 2, logs, ref, 5)


@pytest.mark.gpu
def test_refused_step_does_not_write_a_published_log_buffer():
    """Steps 0-2 with log buffers L0-L2; after step 1 has published L0 the caller reuses it (sentinel).  A refused step 3,
    then step 3 again without fan-out: L0 keeps the sentinel (the refused call must not move the handle's counter, or the
    retry reads as a counter jump and flushes step 3's accumulator row through L0's stale pointer), and L2 receives the
    oracle's row of step 2 (the jump would also re-arm the block and drop it)."""
    _need_gpu()
    from wheeledlab_b200._lib import WlError
    sim, orc = _handle()
    logs, ref = [_nan_log() for _ in range(4)], {}
    ref[0] = _checked_step(sim, orc, 0, logs[0])
    ref[1] = _checked_step(sim, orc, 1, logs[1])
    torch.cuda.synchronize()
    _check_log(logs[0].cpu().numpy(), ref[0], "L0 as published by step 1")
    logs[0].view(torch.uint8).fill_(SENT)
    ref[2] = _checked_step(sim, orc, 2, logs[2])
    ar = _Arena(sim.num_envs, 1, 2, 0)
    sim.set_kernel_variant(4)
    sim.set_peer_fanout([ar.delta(1)])
    with pytest.raises(WlError):
        sim.step(_synth(sim, 3), 3, out=ar.outputs(0), log=logs[3])
    sim.set_peer_fanout([])
    sim.set_kernel_variant(0)
    ref[3] = _checked_step(sim, orc, 3, logs[3])
    sim.flush_log()
    torch.cuda.synchronize()
    assert bool((logs[0].view(torch.uint8) == SENT).all()), "the retried step wrote the published log buffer of step 0"
    _check_log(logs[2].cpu().numpy(), ref[2], "L2")
    _check_log(logs[3].cpu().numpy(), ref[3], "L3")
    _untouched([ar.buf], "refused step")


@pytest.mark.gpu
def test_peer_deltas_must_be_multiples_of_16():
    """The packed rows are 16-byte stores at pointer + delta.  Only the setters are called: no step runs on this handle."""
    _need_gpu()
    from wheeledlab_b200._lib import WlError
    sim, _ = _handle(n=64)
    try:
        for bad in ([8], [4096, -24], [4], [4096, 4096 + 1]):
            with pytest.raises(WlError, match="multiple of 16"):
                sim.set_peer_fanout(bad)
            sim.set_peer_fanout([])
        sim.set_peer_fanout([4096])
        with pytest.raises(WlError, match="multiple of 16"):
            sim.set_multicast_fanout((1 << 30) + 8)
        sim.set_peer_fanout([-4096, 4096 * 3, 16])            # multiples of 16, either sign: accepted
    finally:
        sim.set_multicast_fanout(0)
        sim.set_peer_fanout([])


@pytest.mark.gpu
def test_multicast_delta_needs_peer_deltas():
    """The rows multicast cannot carry go peer by peer, so a multicast delta without peer deltas is refused, and clearing the
    peers clears it.  Only the setters are called: no step runs while a multicast delta may be set."""
    _need_gpu()
    from wheeledlab_b200._lib import WlError
    sim, _ = _handle(n=64)
    mc = 1 << 30
    try:
        with pytest.raises(WlError, match="peer"):
            sim.set_multicast_fanout(mc)
        sim.set_multicast_fanout(0)                           # switching it off is always accepted
        sim.set_peer_fanout([4096])
        sim.set_multicast_fanout(mc)                          # with peers: accepted
        sim.set_peer_fanout([])                               # clears both
        with pytest.raises(WlError, match="peer"):
            sim.set_multicast_fanout(mc)
    finally:
        sim.set_multicast_fanout(0)
        sim.set_peer_fanout([])


@pytest.mark.gpu
def test_fanout_setters_refuse_nine_peers_and_other_tasks():
    """At most WL_MAX_PEERS = 8 deltas; Drift-family tasks only (the other tasks' observation rows are written by kernels
    without a fan-out).  Then the handle keeps matching the oracle."""
    _need_gpu()
    wl = _wl()
    from wheeledlab_b200._lib import WlError
    sim, orc = _handle()
    with pytest.raises(WlError):
        sim.set_peer_fanout([4096 * (k + 1) for k in range(9)])
    vis = wl.WheeledSim(wl.visual_task(num_envs=32, seed=1), DEV)
    with pytest.raises(WlError, match="Drift"):
        vis.set_peer_fanout([4096])
    with pytest.raises(WlError, match="Drift"):
        vis.set_multicast_fanout(4096)
    vis.set_peer_fanout([])
    for t in range(3):
        _checked_step(sim, orc, t)
    assert _launch_info(sim)[:3:2] == (8, 1)


