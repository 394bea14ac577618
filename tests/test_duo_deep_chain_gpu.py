"""Deep-chained duo steps: a chained duo step whose recent predecessors are all of other env sets triggers the next launch at
entry and waits for the grid before it only at its aux warp's and janitor's last instruction, so several steps of different
env sets run at once (wl_step_duo_kernel, duo_chain_mode, DESIGN.md 6e).  These tests step C + 1 env sets -- 4096, a ragged
1 001 and C - 1 sets of 8 envs -- in round-robin groups whose sets recur at distance 1, 2, 3, H, H + 1, C and C + 1, with
wl_reset, wl_observe, wl_act_step and (eagerly) the staged step in between, past the 250-step curriculum boundary, eagerly,
in one CUDA graph and with every step kernel PDL-launched (WL_PDL=1, child process).  Every output, every extras["log"] row,
the final state and the weights must equal those of thread-per-env sims stepped one launch at a time, and each handle's
chained and deep counts must be what a restatement of the host's rule gives.  Torch copies and an event queued right after
a deep chain of C grids must see every set's final rows."""
import os
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent
if __name__ == "__main__":                                  # the WL_PDL=1 child of test_deep_chains_with_pdl_everywhere
    sys.path[:0] = [str(ROOT), str(ROOT / "tests")]

torch = pytest.importorskip("torch")

from test_duo_chained_gpu import _bits, _blob, _buffers, _reset_ids, _spec   # noqa: E402

H, C = 4, 32                                                # WL_DEEP_DISTINCT, WL_DEEP_CAP (wl_api.cu)
SIZES = (4096, 1001) + (8,) * (C - 1)                       # C + 1 env sets
PERIODS = (2, 3, H, H + 1, C, C + 1)
ROUNDS = 44                                                 # per period: 264 steps of every set, past t = 250
DEV = "cuda:0"


def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


def _script(graph):
    """[(op, env set, step counter)]: for each period p the sets are cut into groups of p (the last one shorter, down to a
    single set stepped back to back), and each group is stepped round-robin ROUNDS times.  Every 97th step is an act step
    (after an observe of its set), eagerly every 89th a staged step; every 61st step is followed by a reset of the group's
    first set and an observe of its last."""
    ns = len(SIZES)
    ops, t, k = [("observe", 0, 0), ("act", 0, 0)], [1] + [0] * (ns - 1), 0
    for p in PERIODS:
        for g in [list(range(i, min(i + p, ns))) for i in range(0, ns, p)]:
            for _ in range(ROUNDS):
                for s in g:
                    k += 1
                    if k % 97 == 0:
                        ops.append(("observe", s, t[s])); ops.append(("act", s, t[s]))
                    elif not graph and k % 89 == 0:
                        ops.append(("staged", s, t[s]))
                    else:
                        ops.append(("step", s, t[s]))
                    t[s] += 1
                    if k % 61 == 0:
                        ops.append(("reset", g[0], t[g[0]])); ops.append(("observe", g[-1], t[g[-1]]))
    return ops, t


def _modes(ops):
    """How each plain duo step runs, restating duo_chain_mode: chained ("shallow" or "deep") when its set is not in the
    in-flight suffix (the sets stepped since, and including, the last step that was not deep); deep when, in addition, the
    last H duo steps and this one are of distinct sets and the suffix with it is shorter than C.  Act and staged steps
    clear the record; resets and observes do not trigger and leave it."""
    suffix, recent, out = [], [], []
    for op, s, _ in ops:
        if op in ("act", "staged"):
            suffix, recent = [], []
        elif op == "step":
            mode = "none"
            if suffix and s not in suffix:
                distinct = len(set(recent + [s])) == len(recent) + 1
                mode = "deep" if distinct and len(suffix) + 1 < C else "shallow"
            suffix = suffix + [s] if mode == "deep" else [s]
            recent = ([s] + recent)[:H]
            out.append((s, mode))
    return out


def _counts(ops):
    m = _modes(ops)
    chained = [sum(1 for s, x in m if s == i and x != "none") for i in range(len(SIZES))]
    deep = [sum(1 for s, x in m if s == i and x == "deep") for i in range(len(SIZES))]
    return chained, deep


def _run(graph):
    import wheeledlab_b200 as wl
    from wheeledlab_b200.policy import act_step
    sims = [wl.WheeledSim(_spec(n, 60 + i), DEV) for i, n in enumerate(SIZES)]
    for s in sims:
        s.startup(); s.reset(None, 0)
    ops, t_end = _script(graph)
    acts = [torch.stack([s.synth_actions(t) for t in range(te)]) for s, te in zip(sims, t_end)]
    bufs, blob = _buffers(ops, sims, acts), _blob(DEV)
    ids = [_reset_ids(s.num_envs) for s in sims]
    if graph:                                                 # cudaFuncSetAttribute of the act-step kernel, outside the capture
        w = wl.WheeledSim(_spec(8, 1), DEV); w.startup(); w.reset(None, 0)
        f32 = lambda *sh: torch.zeros(sh, device=DEV)
        act_step(w, f32(8, 14), blob, f32(8, 2), f32(8, 2), f32(8), f32(8),
                 (f32(8, 14), f32(8), torch.zeros(8, dtype=torch.uint8, device=DEV), torch.zeros(8, dtype=torch.uint8, device=DEV)), None, 0)

    def body():
        obs_in = None
        for (op, s, t), b in zip(ops, bufs):
            sim = sims[s]
            c = wl.WheeledSim.device_counter_plus(t) if graph else t
            out = (b.get("obs"), b.get("rew"), b.get("term"), b.get("trunc"))
            if op == "step":
                sim.step(b["act"], c, out=out, log=b["log"])
            elif op == "reset":
                sim.reset(ids[s], t)
            elif op == "observe":
                obs_in = sim.observe(t, 1, out=b["obs"])
            elif op == "act":
                act_step(sim, obs_in, blob, b["act"], b["mean"], b["lp"], b["val"], out, b["log"], c)
            elif op == "staged":
                sim.step_stage_a(b["act"], t, rew=b["rew"], term_bits=b["bits"])
                sim.step_stage_b(b["bits"], t, out=(b["obs"], b["term"], b["trunc"]), log=b["log"])
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
    rec = {f"state{i}": s.groups.cpu().numpy() for i, s in enumerate(sims)}
    rec["chained"] = np.array([s.chained_step_count for s in sims])
    rec["deep"] = np.array([s.deep_step_count for s in sims])
    rec.update({f"weights{i}": s.rew_weight.cpu().numpy() for i, s in enumerate(sims)})
    for k, b in enumerate(bufs):
        for f, x in b.items():
            if f not in ("mean", "lp", "val", "bits"):
                rec[f"{k}_{f}"] = x.cpu().numpy()
    return rec


def _check(rec, what, graph):
    import wheeledlab_b200 as wl
    ops, _ = _script(graph)
    chained, deep = _counts(ops)
    assert sum(deep) > 1000 and rec["chained"].tolist() == chained and rec["deep"].tolist() == deep, \
        f"{what}: chained {rec['chained'].tolist()} / deep {rec['deep'].tolist()}, expected {chained} / {deep}"
    sims = [wl.WheeledSim(_spec(n, 60 + i), DEV) for i, n in enumerate(SIZES)]
    w0 = []
    for s in sims:
        s.set_kernel_variant(1); s.startup(); s.reset(None, 0); w0.append(s.rew_weight.cpu().numpy())
    for k, (op, s, t) in enumerate(ops):
        sim, where = sims[s], f"{what}: {op} #{k} of set {s} ({SIZES[s]} envs) at t={t}"
        if op == "reset":
            sim.reset(_reset_ids(sim.num_envs), t)
        elif op == "observe":
            assert np.array_equal(_bits(rec[f"{k}_obs"]), _bits(sim.observe(t, 1).cpu().numpy())), f"{where}: obs differs"
        else:
            log = torch.zeros(16, device=DEV)
            obs, rew, term, trunc = sim.step(torch.from_numpy(rec[f"{k}_act"]).to(DEV), t, log=log)
            sim.flush_log()
            assert np.array_equal(term.cpu().numpy(), rec[f"{k}_term"]) and np.array_equal(trunc.cpu().numpy(), rec[f"{k}_trunc"]), \
                f"{where}: done masks differ"
            assert np.array_equal(_bits(rew.cpu().numpy()), _bits(rec[f"{k}_rew"])), f"{where}: reward differs"
            assert np.array_equal(_bits(obs.cpu().numpy()), _bits(rec[f"{k}_obs"])), f"{where}: obs differs"
            lg, got = log.cpu().numpy(), rec[f"{k}_log"]
            assert np.allclose(got[:8], lg[:8], rtol=1e-5, atol=1e-4), f"{where}: episode-log sums differ"      # float atomics
            assert np.array_equal(got[8:11], lg[8:11]), f"{where}: episode-log counts differ"
    moved = []
    for i, s in enumerate(sims):
        assert np.array_equal(_bits(rec[f"state{i}"]), _bits(s.groups.cpu().numpy())), f"{what}: final state of set {i} differs"
        w = s.rew_weight.cpu().numpy()
        assert np.array_equal(_bits(rec[f"weights{i}"]), _bits(w)), f"{what}: reward weights of set {i} differ"
        moved += [i] if not np.array_equal(w, w0[i]) else []
    # (the boundary moves a set's weights only if one of its envs finished at t = 249: always so at 4 096 and 1 001 envs,
    # not in every 8-env set, whose envs the script resets and pushes off the track)
    assert {0, 1} <= set(moved), f"{what}: the curriculum boundary moved the weights of sets {moved} only"


def test_rule_restatement_covers_every_mode():
    """(No GPU.) The script reaches all three modes; two sets stepped round-robin settle on shallow steps (the two-grid
    protocol) once the last H steps show the recurrence, and H + 1 sets settle on deep steps cut by the recurring set."""
    for graph in (False, True):
        assert {"none", "shallow", "deep"} <= {m for _, m in _modes(_script(graph)[0])}
    two = [m for _, m in _modes([("step", k % 2, k // 2) for k in range(40)])]
    assert two == ["none", "deep", "none"] + ["shallow"] * 37
    five = [m for _, m in _modes([("step", k % (H + 1), k // (H + 1)) for k in range(40)])]
    assert five == (["none"] + ["deep"] * H) * 8


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["eager", "graph"])
def test_deep_chains_match_thread_per_env(mode):
    _need_gpu()
    _check(_run(mode == "graph"), mode, mode == "graph")


@pytest.mark.gpu
def test_deep_chains_with_pdl_everywhere(tmp_path):
    """The same sequences with WL_PDL=1: the act-step and staged kernels between two duo steps are PDL-launched too and
    trigger at entry.  The flag is read when the library loads: a child process runs the chained side."""
    _need_gpu()
    env = dict(os.environ, WL_PDL="1")
    r = subprocess.run([sys.executable, str(Path(__file__).resolve()), str(tmp_path)], env=env, capture_output=True, text=True,
                       timeout=1500, cwd=str(ROOT))
    assert r.returncode == 0, r.stderr[-3000:]
    for mode in ("eager", "graph"):
        with np.load(tmp_path / f"{mode}.npz") as z:
            _check({k: z[k] for k in z.files}, f"WL_PDL=1 {mode}", mode == "graph")


@pytest.mark.gpu
def test_copies_and_event_after_a_deep_chain_see_final_rows():
    """C sets (4096, 1 001 and 8-env sets) stepped once each per round, so that all but about one step in C run deep;
    right after each round, torch copies of every set's outputs on the same stream, and copies on a
    side stream that waits only for an event recorded after the round.  The output buffers are reused every round, so a
    copy that ran before its step had completed would hold the previous round's rows (or a partly written one)."""
    _need_gpu()
    import wheeledlab_b200 as wl
    sizes, K = SIZES[:C], 12
    mk = lambda: [wl.WheeledSim(_spec(n, 80 + i), DEV) for i, n in enumerate(sizes)]
    sims, refs = mk(), mk()
    for s in refs:
        s.set_kernel_variant(1)
    for s in sims + refs:
        s.startup(); s.reset(None, 0)
    acts = [torch.stack([s.synth_actions(t) for t in range(K)]) for s in sims]
    outs = [(torch.empty((n, 14), device=DEV), torch.empty(n, device=DEV), torch.empty(n, dtype=torch.uint8, device=DEV),
             torch.empty(n, dtype=torch.uint8, device=DEV)) for n in sizes]
    side = torch.cuda.Stream()
    same, evented = [], []
    for t in range(K):
        for s, a, o in zip(sims, acts, outs):
            s.step(a[t], t, out=o)
        ev = torch.cuda.Event()
        ev.record()
        same.append([tuple(x.clone() for x in o) for o in outs])
        with torch.cuda.stream(side):
            side.wait_event(ev)
            evented.append([tuple(x.clone() for x in o) for o in outs])
        torch.cuda.current_stream().wait_stream(side)          # (the next round reuses the buffers the side stream reads)
    torch.cuda.synchronize()
    ops = [("step", i, t) for t in range(K) for i in range(len(sizes))]
    exp = [sum(1 for s, m in _modes(ops) if s == i and m == "deep") for i in range(len(sizes))]
    assert [s.deep_step_count for s in sims] == exp and sum(exp) >= (K - 1) * (C - 1), [s.deep_step_count for s in sims]
    for t in range(K):
        for i, r in enumerate(refs):
            got = r.step(acts[i][t], t)
            for name, a, b, c in zip(("obs", "rew", "terminated", "truncated"), got, same[t][i], evented[t][i]):
                assert torch.equal(a, b), f"round {t}, set {i}: the copy of {name} is not the step's final output"
                assert torch.equal(a, c), f"round {t}, set {i}: the copy of {name} after the event is not final"


if __name__ == "__main__":
    dst = Path(sys.argv[1])
    for m in ("eager", "graph"):
        np.savez(dst / f"{m}.npz", **_run(m == "graph"))
