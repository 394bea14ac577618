"""The Drift-family duo step kernel (wl_step_duo_kernel) against the CPU oracle across the config space it special-cases.

- The step-spec matrix: each shipped spec (RWD `drift`, 4WD `hound_4wd`) with one spec field moved at a time runs the generic
  body (K = 0); the shipped and lowered reference cfgs run the two specialised instantiations.  wl_step_launch_info says
  which one ran, so a config that drifts off its spec fails here instead of silently losing the specialised path.
- Launch geometries: ragged CTAs, the spacer-warp cut-off, the hand-over to the thread-per-env kernel and its block sizes.
- Kernels interleaved on one handle and one stream without host syncs (the duo kernel triggers its dependents before its
  last stores), eagerly, in a CUDA graph, and with every step kernel PDL-launched (WL_PDL=1, child process).

Every comparison is bit for bit: obs, reward and done masks every step, the full state and the reward weights at the end; the
episode-log counts exactly and its sums (float atomics: order-dependent) to rtol 1e-5.  The last test runs on the CPU: every
deviation of the matrix changes the oracle's trajectory, so the GPU matrix never compares two runs of a field the dynamics
ignore."""
import ctypes as C
import math
import os
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent
if __name__ == "__main__":                                  # the WL_PDL=1 child of test_interleaved_kernels_with_pdl_everywhere
    sys.path[:0] = [str(ROOT), str(ROOT / "tests")]

import oracle_lib as O  # noqa: E402

torch = pytest.importorskip("torch")

BLOBS = ROOT / "tests" / "golden" / "cfg_blobs"
DRIFT_SIM_DT = 0.005                                        # drift_task's sim_dt in Python doubles (max_episode_length is ceil'd on it)


def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


def _launch_info(sim):
    """(variant, spec key, specialised, threads per CTA) of the most recent wl_step on the handle."""
    import wheeledlab_b200 as wl
    v, k, s, th = C.c_int32(), C.c_uint32(), C.c_int32(), C.c_int32()
    wl._lib.check(wl.lib.wl_step_launch_info(sim._h, C.byref(v), C.byref(k), C.byref(s), C.byref(th)), "wl_step_launch_info")
    return v.value, k.value, s.value, th.value


# ---- configs ---------------------------------------------------------------------------------------------------------
def _decimation(d):
    def f(cfg):
        cfg.decimation = d
        cfg.max_episode_length = math.ceil(float(cfg.episode_length_s) / (DRIFT_SIM_DT * d))     # as drift_task computes it
    return f


def _substeps(s):
    def f(cfg):
        cfg.substeps = s
    return f


def _no_corruption(cfg):
    cfg.enable_corruption = 0


def _reverse(cfg):
    cfg.no_reverse = 0


def _wheel_mass_dr(cfg):
    """Base and wheel masses drawn absolutely, as visual_task(randomize=True) does (the wheel-inertia group WL_G_PIW)."""
    cfg.dr_mass_mode, cfg.dr_wheel_mass_enable = 1, 1
    cfg.dr_mass_add[0], cfg.dr_mass_add[1] = 1.0, 3.0
    cfg.dr_wheel_mass[0], cfg.dr_wheel_mass[1] = 0.01, 0.3


def _all(cfg):
    for f in (_no_corruption, _reverse, _wheel_mass_dr, _decimation(2), _substeps(3)):
        f(cfg)


DEVIATIONS = {
    "no_corruption": _no_corruption, "reverse": _reverse, "wheel_mass_dr": _wheel_mass_dr,
    "decimation1": _decimation(1), "decimation2": _decimation(2), "decimation10": _decimation(10),
    "substeps2": _substeps(2), "substeps3": _substeps(3), "all": _all,
}
WIDE = {"reverse", "all"}                                   # N(0, 2) actions: negative throttle reaches the no_reverse branch
SPECIALISED = ["drift", "hound_4wd", "f1tenth_drift",       # make_task names, then the lowered reference cfgs
               "Isaac-MushrDriftRL-v0.ref", "Isaac-MushrDriftRL-v0.play.ref", "Isaac-F1TenthDriftRL-v0.ref"]


def _spec(name, n, seed=11, deviation=None):
    """A Drift-family TaskSpec with `n` envs and every curriculum term firing at each episode boundary."""
    import wheeledlab_b200 as wl
    if name.endswith(".ref"):
        spec = wl.drift_task(num_envs=n, seed=seed)
        raw = (BLOBS / f"{name}.bin").read_bytes()
        assert len(raw) == C.sizeof(spec.cfg)
        C.memmove(C.addressof(spec.cfg), raw, len(raw))      # the lowered cfg (same struct as oracle_lib.cfg_from_blob reads)
        spec.cfg.num_envs = n
    else:
        spec = wl.make_task(name, num_envs=n, seed=seed)
    for k in range(spec.cfg.curr_n):
        spec.cfg.curr_every[k] = 1
    if deviation is not None:
        DEVIATIONS[deviation](spec.cfg)
    return spec


def _spec_key(name):
    """The step-spec key wl_create derives for a shipped task's config."""
    import wheeledlab_b200 as wl
    return _launch_info(wl.WheeledSim(_spec(name, 8), "cuda:0"))[1]


def _synth(sim, t):
    return sim.synth_actions(t, dist=t % 2)


def _wide_actions(sim, t):
    g = torch.Generator(device="cuda").manual_seed(1000 + t)
    return torch.randn((sim.num_envs, 2), generator=g, device="cuda") * 2.0


def _check_log(got, lg, what):
    assert np.allclose(got[:8], lg[:8], rtol=1e-5, atol=1e-4), f"{what}: episode-log sums differ"      # float atomics
    assert np.array_equal(got[8:11], lg[8:11].astype(np.float32)), f"{what}: episode-log counts differ"


def _check_step(got, ref, what):
    obs, rew, term, trunc = (x.cpu().numpy() if torch.is_tensor(x) else x for x in got)
    o_obs, o_rew, o_term, o_trunc = ref
    assert np.array_equal(term, o_term) and np.array_equal(trunc, o_trunc), f"{what}: done masks differ"
    assert np.array_equal(_bits(rew), _bits(o_rew)), f"{what}: reward differs"
    assert np.array_equal(_bits(obs), _bits(o_obs)), f"{what}: obs differs"
    return int((o_term | o_trunc).sum())


def _oracle_traj(spec, steps, action_fn=_synth, threads=8):
    """Default kernel variant vs the oracle, every output every step, state and weights at the end.  Returns the sim (for
    wl_step_launch_info) and the oracle."""
    import wheeledlab_b200 as wl
    sim = wl.WheeledSim(spec, "cuda:0"); sim.startup(); sim.reset(None, 0)
    orc = O.Oracle(spec.cfg, threads=threads); orc.startup(); orc.reset(None, 0)
    w0 = sim.rew_weight.cpu().numpy().copy()
    n_done = 0
    for t in range(steps):
        act = action_fn(sim, t)
        log = torch.empty(16, device="cuda")
        out = sim.step(act, t, log=log)
        sim.flush_log()                                       # the row of step t is published by the next launch on the handle
        n_done += _check_step(out, orc.step(act.cpu().numpy(), t), f"step {t}")
        _check_log(log.cpu().numpy(), orc.log(), f"step {t}")
    assert np.array_equal(_bits(sim.groups.cpu().numpy()), _bits(orc.export_state())), "final state differs"
    w = sim.rew_weight.cpu().numpy()
    assert np.array_equal(_bits(w), _bits(orc.weights())), "reward weights differ"
    if spec.cfg.term_enable:
        assert n_done > 0, "trajectory too short to exercise the auto-reset"
    else:                                                     # (the lowered play cfg has no termination term at all)
        assert n_done == 0, "an env reset with every termination term off"
    if spec.cfg.curr_n > 0 and steps > spec.cfg.max_episode_length:
        assert not np.array_equal(w, w0), "the curriculum boundary did not move the weights"
    return sim, orc


# ---- 2. the step-spec matrix -----------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("n,steps", [(4096, 300), (333, 120)])
@pytest.mark.parametrize("deviation", list(DEVIATIONS))
@pytest.mark.parametrize("base", ["drift", "hound_4wd"])
def test_generic_duo_body_matches_oracle(base, deviation, n, steps):
    """One step-spec field moved off a shipped spec: the duo kernel's generic body (K = 0) runs it, reading at run time what
    the specialised instantiations fold.  4096 envs: one CTA per 8 envs with the spacer warp; 333: a ragged last CTA."""
    _need_gpu()
    spec = _spec(base, n, deviation=deviation)
    sim, orc = _oracle_traj(spec, steps, _wide_actions if deviation in WIDE else _synth)
    variant, key, specialised, threads = _launch_info(sim)
    assert (variant, specialised, threads) == (8, 0, 96), (variant, specialised, threads)
    assert key != _spec_key(base), "the deviation did not change the step-spec key"
    if deviation == "no_corruption":                          # no noise: every observe() call gives the same rows
        a, b = sim.observe(steps, 0).cpu().numpy(), sim.observe(steps, 1).cpu().numpy()
        assert np.array_equal(_bits(a), _bits(b)) and np.array_equal(_bits(a), _bits(orc.observe(steps, 0)))


@pytest.mark.gpu
@pytest.mark.parametrize("n,steps", [(4096, 300), (333, 120)])
@pytest.mark.parametrize("name", SPECIALISED)
def test_specialised_duo_instantiation_matches_oracle(name, n, steps):
    """The shipped Drift-family tasks and the lowered reference Drift / F1Tenth train and play cfgs (the reference registers
    no F1Tenth play cfg) run one of the two spec instantiations (SPEC_DRIFT_RWD / SPEC_DRIFT_4WD in wl_api.cu).  The play
    cfg turns every termination term off, so its envs never reset; the train cfg runs the reset path on the same key."""
    _need_gpu()
    sim, _ = _oracle_traj(_spec(name, n), steps)
    variant, key, specialised, threads = _launch_info(sim)
    assert (variant, specialised, threads) == (8, 1, 96), (name, variant, specialised, threads)
    assert key == _spec_key("drift" if int(sim.cfg.action_kind) == 1 else "hound_4wd"), name


# ---- 3. launch geometries --------------------------------------------------------------------------------------------
def _geometry_spec(n):
    """The `drift` spec with 25-step episodes (not a step-spec field): every CTA, ragged ones included, takes the reset path
    within the run."""
    spec = _spec("drift", n, seed=3)
    spec.cfg.max_episode_length = 25
    return spec


def _geometry_run(n, steps=40):
    sim, _ = _oracle_traj(_geometry_spec(n), steps)
    return _launch_info(sim)


@pytest.mark.gpu
@pytest.mark.parametrize("n,variant,threads", [
    (1, 8, 96), (7, 8, 96), (9, 8, 96),                       # one ragged CTA; a full one + one env
    (4095, 8, 96),                                            # ragged last CTA with the spacer warp
    (8197, 8, 64),                                            # ragged, past the spacer cut-off: 2-warp CTAs
    (32 * 132 * 4 * 2, 8, 64),                                # 33 792 = WL_QUAD_MAX_ENVS: the last duo-kernel size
    (32 * 132 * 4 * 2 + 1, 1, 64),                            # the first thread-per-env size (pick_block: 64)
    (132 * 128 * 4, 1, 128),                                  # 67 584: pick_block's 128-thread CTAs
])
def test_launch_geometry_matches_oracle(n, variant, threads):
    _need_gpu()
    v, _, specialised, th = _geometry_run(n, steps=40 if n < 30000 else 30)
    assert (v, th) == (variant, threads), (n, v, th)
    assert specialised == (1 if variant == 8 else 0)


@pytest.mark.gpu
def test_spacer_warp_cutoff_both_sides_match_oracle():
    """duo_block keeps the spacer warp while the occupancy query says every CTA is resident at once.  The cut-off is read
    from wl_step_launch_info (the first N launched with 64 threads per CTA) and the sizes around it are run."""
    _need_gpu()
    import wheeledlab_b200 as wl

    def threads_at(n):
        sim = wl.WheeledSim(_spec("drift", n), "cuda:0"); sim.startup(); sim.reset(None, 0)
        sim.step(torch.zeros((n, 2), device="cuda"), 0)
        return _launch_info(sim)[3]

    lo, hi = 4096, 8192
    assert threads_at(lo) == 96 and threads_at(hi) == 64
    while hi - lo > 1:
        mid = (lo + hi) // 2
        lo, hi = (mid, hi) if threads_at(mid) == 96 else (lo, mid)
    print(f"spacer cut-off: {hi} envs (last with the spacer warp: {lo})")
    seen = [_geometry_run(m)[3] for m in (hi - 1, hi, hi + 1)]
    assert seen == [96, 64, 64], seen


# ---- 4. kernels interleaved on one handle ----------------------------------------------------------------------------
ROLL_K = 5


def _script(graph):
    """[(op, step counter)] until the counter passes 250.  The graph form holds only operations that take the device counter
    (reset and observe take a counter only as a key of their draws): no staged step and no rollout."""
    ops, t = [], 0
    while t <= 250:
        ops.append(("step", t)); t += 1
        ops.append(("reset", t)); ops.append(("observe", t))
        if not graph:
            ops.append(("staged", t)); t += 1
        ops.append(("act", t)); t += 1
        if not graph and (t + ROLL_K - 1) // 250 == t // 250:          # a rollout may not cross a curriculum boundary
            ops.append(("rollout", t)); t += ROLL_K
        ops.append(("step", t)); t += 1
    return ops, t


def _reset_ids(n):
    return np.array(sorted({0, 3, n // 2, n - 1}), np.int64)


def _interleave_spec(n):
    return _spec("drift", n, seed=29)


def _run_interleaved(n, graph):
    """The sequence of _script on one handle and one stream, no host sync until the end.  Returns every output as numpy."""
    import wheeledlab_b200 as wl
    from wheeledlab_b200.distributed import RolloutSlab
    from wheeledlab_b200.policy import act_step, pack_actor_critic
    dev = "cuda:0"
    sim = wl.WheeledSim(_interleave_spec(n), dev); sim.startup(); sim.reset(None, 0)
    ops, t_end = _script(graph)
    acts = torch.stack([sim.synth_actions(t) for t in range(t_end)])
    torch.manual_seed(0)
    mk = lambda out: torch.nn.Sequential(torch.nn.Linear(14, 64), torch.nn.ELU(), torch.nn.Linear(64, 64), torch.nn.ELU(), torch.nn.Linear(64, out)).to(dev)
    blob = pack_actor_critic(mk(2), mk(1), torch.tensor([0.7, 1.3], device=dev), 14, dev)
    ids = torch.from_numpy(_reset_ids(n)).to(dev)
    f32 = lambda *s: torch.empty(s, dtype=torch.float32, device=dev)
    u8 = lambda *s: torch.empty(s, dtype=torch.uint8, device=dev)
    bufs = []
    for op, t in ops:
        b = {}
        if op in ("step", "staged", "act"):
            b = {"obs": f32(n, 14), "rew": f32(n), "term": u8(n), "trunc": u8(n), "log": torch.zeros(16, device=dev)}
            b["act"] = acts[t] if op != "act" else f32(n, 2)
        if op == "act":
            b.update(mean=f32(n, 2), lp=f32(n), val=f32(n))
        if op == "staged":
            b.update(bits=u8(n))
        if op == "observe":
            b = {"obs": f32(n, 14)}
        if op == "rollout":
            b = {"slab": RolloutSlab(ROLL_K, n, 14, 2, dev), "log": torch.zeros((ROLL_K, 16), device=dev)}
        bufs.append(b)
    if graph:                                                 # cudaFuncSetAttribute of the act-step kernel, outside the capture
        w = wl.WheeledSim(_interleave_spec(8), dev); w.startup(); w.reset(None, 0)
        act_step(w, f32(8, 14).zero_(), blob, f32(8, 2), f32(8, 2), f32(8), f32(8), (f32(8, 14), f32(8), u8(8), u8(8)), None, 0)
    w0 = sim.rew_weight.clone()

    def body():
        obs_in = None                                         # (every act op follows an observe op)
        for (op, t), b in zip(ops, bufs):
            c = wl.WheeledSim.device_counter_plus(t) if graph else t
            out = (b.get("obs"), b.get("rew"), b.get("term"), b.get("trunc"))
            if op == "step":
                sim.step(b["act"], c, out=out, log=b["log"])
            elif op == "reset":
                sim.reset(ids, t)
            elif op == "observe":
                obs_in = sim.observe(t, 1, out=b["obs"])
            elif op == "staged":
                sim.step_stage_a(b["act"], t, rew=b["rew"], term_bits=b["bits"])
                sim.step_stage_b(b["bits"], t, out=(b["obs"], b["term"], b["trunc"]), log=b["log"])
            elif op == "act":
                act_step(sim, obs_in, blob, b["act"], b["mean"], b["lp"], b["val"], out, b["log"], c)
            elif op == "rollout":
                sim.rollout(ROLL_K, t, b["slab"], b["log"])
        if graph:
            sim.advance_counter(t_end)

    sim.set_step_counter(0)
    if graph:
        g, s = torch.cuda.CUDAGraph(), torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            with torch.cuda.graph(g, stream=s):
                body()
        torch.cuda.current_stream().wait_stream(s)
        sim.set_step_counter(0)                               # (capture moved the host mirror only)
        g.replay()
    else:
        body()
    sim.flush_log()
    torch.cuda.synchronize()
    rec = {"state": sim.groups.cpu().numpy(), "weights": sim.rew_weight.cpu().numpy(), "weights0": w0.cpu().numpy()}
    for k, ((op, _), b) in enumerate(zip(ops, bufs)):
        if op == "rollout":
            sl = b["slab"]
            for f, x in (("act", sl.actions), ("obs", sl.obs), ("rew", sl.rewards), ("term", sl.terminated), ("trunc", sl.truncated), ("log", b["log"])):
                rec[f"{k}_{f}"] = x.cpu().numpy()
        else:
            for f in ("act", "obs", "rew", "term", "trunc", "log"):
                if f in b:
                    rec[f"{k}_{f}"] = b[f].cpu().numpy()
    return rec


def _replay_on_oracle(n, graph, rec):
    spec = _interleave_spec(n)
    orc = O.Oracle(spec.cfg, threads=8); orc.startup(); orc.reset(None, 0)
    ops, _ = _script(graph)
    n_done = 0
    for k, (op, t) in enumerate(ops):
        what = f"{'graph' if graph else 'eager'} n={n}: {op} #{k} at t={t}"
        if op == "reset":
            orc.reset(_reset_ids(n), t)
        elif op == "observe":
            assert np.array_equal(_bits(rec[f"{k}_obs"]), _bits(orc.observe(t, 1))), f"{what}: obs differs"
        elif op == "rollout":
            for j in range(ROLL_K):
                got = tuple(rec[f"{k}_{f}"][j] for f in ("obs", "rew", "term", "trunc"))
                n_done += _check_step(got, orc.step(rec[f"{k}_act"][j], t + j), f"{what}+{j}")
                _check_log(rec[f"{k}_log"][j], orc.log(), f"{what}+{j}")
        else:
            got = tuple(rec[f"{k}_{f}"] for f in ("obs", "rew", "term", "trunc"))
            n_done += _check_step(got, orc.step(rec[f"{k}_act"], t), what)
            _check_log(rec[f"{k}_log"], orc.log(), what)
    assert np.array_equal(_bits(rec["state"]), _bits(orc.export_state())), f"n={n}: final state differs"
    assert np.array_equal(_bits(rec["weights"]), _bits(orc.weights())), f"n={n}: reward weights differ"
    assert not np.array_equal(rec["weights"], rec["weights0"]), "the curriculum boundary did not move the weights"
    assert n_done > 0, "no auto-reset in the sequence"


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["eager", "graph"])
@pytest.mark.parametrize("n", [4096, 333])
def test_interleaved_kernels_on_one_handle_match_oracle(n, mode):
    """duo wl_step, wl_reset of fixed ids, wl_observe, the staged step, wl_act_step (its sampled actions go to the oracle),
    wl_rollout (its in-kernel actions go to the oracle), duo wl_step again, repeated past t = 250 on one stream.  At 333
    envs a step after a rollout often resets no env, so its log row must repeat the rollout's last row with a reset."""
    _need_gpu()
    _replay_on_oracle(n, mode == "graph", _run_interleaved(n, mode == "graph"))


@pytest.mark.gpu
def test_interleaved_kernels_with_pdl_everywhere(tmp_path):
    """The same sequences with WL_PDL=1: the thread, quad and act-step kernels are PDL-launched too, so each one's prologue
    may overlap the kernel before it and its griddepcontrol.wait alone orders its reads.  The flag is read when the library
    loads: a child process runs the device side and the oracle checks its outputs here."""
    _need_gpu()
    env = dict(os.environ, WL_PDL="1")
    r = subprocess.run([sys.executable, str(Path(__file__).resolve()), str(tmp_path)], env=env, capture_output=True, text=True,
                       timeout=900, cwd=str(ROOT))
    assert r.returncode == 0, r.stderr[-3000:]
    for n in (4096, 333):
        for graph in (False, True):
            with np.load(tmp_path / f"{n}_{'graph' if graph else 'eager'}.npz") as z:
                _replay_on_oracle(n, graph, {k: z[k] for k in z.files})


# ---- 5. every deviation is live (CPU) --------------------------------------------------------------------------------
@pytest.mark.parametrize("deviation", list(DEVIATIONS))
@pytest.mark.parametrize("base", ["drift", "hound_4wd"])
def test_every_deviation_changes_the_oracle_trajectory(base, deviation):
    n, steps = 64, 60

    def run(dev):
        spec = _spec(base, n, deviation=dev)
        orc = O.Oracle(spec.cfg); orc.startup(); orc.reset(None, 0)
        rng = np.random.default_rng(5)
        trace = []
        for t in range(steps):
            a = (rng.normal(size=(n, 2)) * 2.0).astype(np.float32) if deviation in WIDE else orc.synth_actions(t, t % 2)
            obs, rew, term, trunc = orc.step(a, t)
            trace += [obs, rew, term, trunc]
        return trace + [orc.export_state()]

    base_run, dev_run = run(None), run(deviation)
    assert any(not np.array_equal(_bits(a) if a.dtype == np.float32 else a, _bits(b) if b.dtype == np.float32 else b)
               for a, b in zip(base_run, dev_run)), f"{base}: {deviation} leaves the trajectory unchanged"


if __name__ == "__main__":
    out = Path(sys.argv[1])
    for n in (4096, 333):
        for graph in (False, True):
            np.savez(out / f"{n}_{'graph' if graph else 'eager'}.npz", **_run_interleaved(n, graph))
