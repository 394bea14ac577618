"""Deep-chained duo steps in CTAs of four env warps and one aux warp (32 envs per CTA, wl_step_duo_deep_kernel, DESIGN.md 6e).

Eleven env sets of 1, 7, 8, 9, 31, 32, 33, 96, 1 001, 4 096 and 8 192 envs -- CTAs with one to four live env warps, ragged
quads and aux lanes past the last env -- are stepped round-robin, so that nearly every step runs deep, past the 250-step
curriculum boundary, with interval pushes, auto-resets and explicit resets, eagerly and in one CUDA graph.  The RWD and 4WD
step specs and one generic config (tanh-bounded Drift) are covered.  Every output, every extras["log"] row, the final state
and the weights must equal those of thread-per-env sims stepped one launch at a time; deep steps must report 160 threads per
CTA, and the other duo steps the width an unchained step of the same set reports."""
import ctypes as C

import numpy as np
import pytest

torch = pytest.importorskip("torch")

from test_duo_deep_chain_gpu import _modes   # noqa: E402

pytestmark = pytest.mark.gpu

SIZES = (1, 7, 8, 9, 31, 32, 33, 96, 1001, 4096, 8192)
ROUNDS = 262                                                # every set steps past t = 250
RESET_EVERY = 41                                            # rounds between explicit resets of one set
DEEP_THREADS = 160
DEV = "cuda:0"


def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


def _spec(task, n, seed):
    import wheeledlab_b200 as wl
    from wheeledlab_b200.tasks import BOUND_TANH
    spec = wl.make_task("drift" if task == "drift_tanh" else task, num_envs=n, seed=seed)
    if task == "drift_tanh":
        spec.cfg.bounding = BOUND_TANH                       # no specialisation has this spec: the generic body runs it
    for k in range(spec.cfg.curr_n):
        spec.cfg.curr_every[k] = 1                           # every term's weight moves at the first boundary (t = 250)
    return spec


def _launch_info(sim):
    """(variant, spec key, specialised, threads per CTA) of the most recent wl_step on the handle."""
    import wheeledlab_b200 as wl
    v, k, s, th = C.c_int32(), C.c_uint32(), C.c_int32(), C.c_int32()
    wl._lib.check(wl.lib.wl_step_launch_info(sim._h, C.byref(v), C.byref(k), C.byref(s), C.byref(th)), "wl_step_launch_info")
    return v.value, k.value, s.value, th.value


def _reset_ids(n):
    return torch.tensor(sorted({0, n // 2, n - 1}), dtype=torch.int64, device=DEV)


def _script():
    """[(op, env set, step counter)]: every round steps each set once in order; every RESET_EVERY-th round ends with a reset
    of one set (resets do not change how the next step runs)."""
    ops, t = [], [0] * len(SIZES)
    for r in range(ROUNDS):
        for s in range(len(SIZES)):
            ops.append(("step", s, t[s]))
            t[s] += 1
        if r % RESET_EVERY == RESET_EVERY - 1:
            s = (r // RESET_EVERY) % len(SIZES)
            ops.append(("reset", s, t[s]))
    return ops, t


def _run(task, graph):
    import wheeledlab_b200 as wl
    sims = [wl.WheeledSim(_spec(task, n, 30 + i), DEV) for i, n in enumerate(SIZES)]
    for s in sims:
        s.startup(); s.reset(None, 0)
    ops, t_end = _script()
    acts = [torch.stack([s.synth_actions(t) for t in range(te)]) for s, te in zip(sims, t_end)]
    f32 = lambda *sh: torch.empty(sh, dtype=torch.float32, device=DEV)
    u8 = lambda *sh: torch.empty(sh, dtype=torch.uint8, device=DEV)
    bufs = [{"obs": f32(sims[s].num_envs, 14), "rew": f32(sims[s].num_envs), "term": u8(sims[s].num_envs),
             "trunc": u8(sims[s].num_envs), "log": torch.zeros(16, device=DEV)} if op == "step" else {} for op, s, _ in ops]
    ids = [_reset_ids(s.num_envs) for s in sims]
    threads = []
    # a thread-per-env step clears the stream's record of duo steps, so that the script's first step runs unchained
    clr = wl.WheeledSim(_spec(task, 1, 99), DEV)
    clr.set_kernel_variant(1); clr.startup(); clr.reset(None, 0)
    clr_act = clr.synth_actions(0)

    def body():
        if not graph:
            clr.step(clr_act, 0)
        for (op, s, t), b in zip(ops, bufs):
            sim = sims[s]
            if op == "step":
                sim.step(acts[s][t], wl.WheeledSim.device_counter_plus(t) if graph else t,
                         out=(b["obs"], b["rew"], b["term"], b["trunc"]), log=b["log"])
                threads.append(_launch_info(sim))
            else:
                sim.reset(ids[s], t)
        if graph:
            for sim, te in zip(sims, t_end):
                sim.advance_counter(te)

    for sim in sims:
        sim.set_step_counter(0)
    if graph:
        g, st = torch.cuda.CUDAGraph(), torch.cuda.Stream()
        st.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(st):
            with torch.cuda.graph(g, stream=st):
                body()
        torch.cuda.current_stream().wait_stream(st)
        for sim in sims:
            sim.set_step_counter(0)
        g.replay()
    else:
        body()
    for sim in sims:
        sim.flush_log()
    torch.cuda.synchronize()
    rec = {"state": [s.groups.cpu().numpy() for s in sims], "weights": [s.rew_weight.cpu().numpy() for s in sims],
           "deep": [s.deep_step_count for s in sims], "launch": threads, "acts": [a.cpu() for a in acts],
           "out": [{k: x.cpu().numpy() for k, x in b.items()} for b in bufs]}
    return rec


def _unchained_width(task, n):
    """threads per CTA of a duo step that runs neither chained nor deep: one that follows a step of its own set"""
    import wheeledlab_b200 as wl
    sim = wl.WheeledSim(_spec(task, n, 1), DEV)
    sim.startup(); sim.reset(None, 0)
    sim.step(sim.synth_actions(0), 0)
    chained = sim.chained_step_count
    sim.step(sim.synth_actions(1), 1)
    torch.cuda.synchronize()
    assert sim.chained_step_count == chained
    return _launch_info(sim)


@pytest.mark.parametrize("task", ["drift", "hound_4wd", "drift_tanh"])
@pytest.mark.parametrize("mode", ["eager", "graph"])
def test_wide_deep_chains_match_thread_per_env(task, mode):
    _need_gpu()
    import wheeledlab_b200 as wl
    graph = mode == "graph"
    rec = _run(task, graph)
    ops, _ = _script()
    modes = _modes(ops)
    steps = [(s, t) for op, s, t in ops if op == "step"]
    assert len(modes) == len(steps) == len(rec["launch"])
    deep = [sum(1 for s, m in modes if s == i and m == "deep") for i in range(len(SIZES))]
    assert rec["deep"] == deep and sum(deep) > 0.9 * len(steps), (rec["deep"], deep)
    widths = {n: _unchained_width(task, n) for n in SIZES}
    for (s, m), (variant, key, specialised, th) in zip(modes, rec["launch"]):
        assert variant == 8 and bool(specialised) == (task != "drift_tanh"), (task, variant, key, specialised)
        expect = DEEP_THREADS if m == "deep" else widths[SIZES[s]][3]
        assert th == expect, f"{task} {mode}: a {m} step of {SIZES[s]} envs reported {th} threads per CTA, expected {expect}"
    assert {w[3] for w in widths.values()} <= {64, 96}, widths

    sims = [wl.WheeledSim(_spec(task, n, 30 + i), DEV) for i, n in enumerate(SIZES)]
    w0 = []
    for s in sims:
        s.set_kernel_variant(1); s.startup(); s.reset(None, 0); w0.append(s.rew_weight.cpu().numpy())
    resets = 0
    for k, (op, s, t) in enumerate(ops):
        sim, where = sims[s], f"{task} {mode}: {op} #{k} of set {s} ({SIZES[s]} envs) at t={t}"
        if op == "reset":
            sim.reset(_reset_ids(sim.num_envs), t)
            continue
        got = rec["out"][k]
        log = torch.zeros(16, device=DEV)
        obs, rew, term, trunc = sim.step(rec["acts"][s][t].to(DEV), t, log=log)
        sim.flush_log()
        term, trunc = term.cpu().numpy(), trunc.cpu().numpy()
        resets += int((term | trunc).sum())
        assert np.array_equal(term, got["term"]) and np.array_equal(trunc, got["trunc"]), f"{where}: done masks differ"
        assert np.array_equal(_bits(rew.cpu().numpy()), _bits(got["rew"])), f"{where}: reward differs"
        assert np.array_equal(_bits(obs.cpu().numpy()), _bits(got["obs"])), f"{where}: obs differs"
        lg = log.cpu().numpy()
        assert np.allclose(got["log"][:8], lg[:8], rtol=1e-5, atol=1e-4), f"{where}: episode-log sums differ"   # float atomics
        assert np.array_equal(got["log"][8:11], lg[8:11]), f"{where}: episode-log counts differ"
    assert resets > 0, f"{task}: no env reset on its own"
    moved = []
    for i, s in enumerate(sims):
        assert np.array_equal(_bits(rec["state"][i]), _bits(s.groups.cpu().numpy())), f"{task} {mode}: final state of set {i} differs"
        w = s.rew_weight.cpu().numpy()
        assert np.array_equal(_bits(rec["weights"][i]), _bits(w)), f"{task} {mode}: reward weights of set {i} differ"
        moved += [i] if not np.array_equal(w, w0[i]) else []
    # (the boundary moves a set's weights only if one of its envs finished at t = 249: the large sets always have one)
    assert {9, 10} <= set(moved), f"{task} {mode}: the curriculum boundary moved the weights of sets {moved} only"
