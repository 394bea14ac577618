"""Chained duo steps: a single-GPU duo step whose stream predecessor is a duo step of ANOTHER env set starts its env CTAs on
entry, without griddepcontrol.wait; its aux warp waits before the episode log, the reward weights and its trigger
(wl_step_duo_kernel, DESIGN.md 6e).  These tests step several env sets on one stream -- 4096 envs, a ragged 1 001 and 8,
round-robin, the smallest also back to back -- with wl_reset, wl_observe and wl_act_step in between, past the 250-step
curriculum boundary, eagerly (with the staged step, wl_rollout and a counter jump too), in one CUDA graph and with every
step kernel PDL-launched (WL_PDL=1, child process).  Every output, every extras["log"] row, the final state and the weights
must equal those of thread-per-env sims stepped through the same sequence one launch at a time; they replace a direct oracle
comparison here, since test_duo_coverage_gpu.py and test_gpu_parity.py hold the thread-per-env kernel to the oracle bit for
bit.  The handles' chained-step counts must be exactly the steps the sequence allows to run chained.  A step's outputs must
also be final for a plain torch kernel queued right after the next env set's step."""
import os
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent
if __name__ == "__main__":                                  # the WL_PDL=1 child of test_round_robin_with_pdl_everywhere
    sys.path[:0] = [str(ROOT), str(ROOT / "tests")]

torch = pytest.importorskip("torch")

SIZES = (4096, 1001, 8)
ROUNDS = 260
DEV = "cuda:0"
ROLL_K = 5


def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


def _spec(n, seed):
    import wheeledlab_b200 as wl
    spec = wl.make_task("drift", num_envs=n, seed=seed)
    for k in range(spec.cfg.curr_n):
        spec.cfg.curr_every[k] = 1                           # every term's weight moves at the first boundary (t = 250)
    return spec


def _reset_ids(n):
    return torch.tensor(sorted({0, 3, n // 2, n - 1}), dtype=torch.int64, device=DEV)


def _script(graph):
    """[(op, env set, step counter)]: each round steps sets 0, 1, 2 and set 2 again; every 4th round resets envs of set 0
    and observes set 1, and every 4th (offset) set 0 takes an act step before its plain step.  Eagerly also: every 6th
    round a staged step of set 1 right after set 0's step (so set 1's step follows a staged step, with set 0's step the
    last duo launch), every 6th (offset) a rollout of set 2 before its steps, and one counter jump of set 1 (the rearm).
    The graph form keeps only operations that take the device counter.  The first ops are an observe and an act step, so
    the chained launches of the sequence do not depend on what ran on the stream before it."""
    ops, t = [("observe", 0, 0), ("act", 0, 0)], [1, 0, 0]
    for r in range(ROUNDS):
        if r % 4 == 3:                                        # (the act step triggers at entry: the step after it waits)
            ops.append(("observe", 0, t[0])); ops.append(("act", 0, t[0])); t[0] += 1
        ops.append(("step", 0, t[0])); t[0] += 1
        if not graph and r % 6 == 2:                          # (the staged kernel triggers at entry: set 1's step waits)
            ops.append(("staged", 1, t[1])); t[1] += 1
        if not graph and r == 100:
            t[1] += 3                                         # counter jump: prep_step re-arms set 1 before its step
        ops.append(("step", 1, t[1])); t[1] += 1
        if not graph and r % 6 == 4 and (t[2] + ROLL_K - 1) // 250 == t[2] // 250:
            ops.append(("rollout", 2, t[2])); t[2] += ROLL_K  # (does not trigger: set 2's step after it runs chained)
        for s in (2, 2):
            ops.append(("step", s, t[s])); t[s] += 1
        if r % 4 == 1:
            ops.append(("reset", 0, t[0])); ops.append(("observe", 1, t[1]))
    return ops, t


def _expected_chained(ops):
    """The duo steps that run chained: the previous op that triggers its dependents (a step, act step or staged step) is a
    plain step of another set.  Resets, observes, rollouts and the rearm do not trigger."""
    prev, n = None, 0
    for op, s, _ in ops:
        if op in ("step", "act", "staged"):
            n += op == "step" and prev is not None and prev[0] == "step" and prev[1] != s
            prev = (op, s)
    return n


def _blob(dev):
    from wheeledlab_b200.policy import pack_actor_critic
    torch.manual_seed(0)
    mk = lambda out: torch.nn.Sequential(torch.nn.Linear(14, 64), torch.nn.ELU(), torch.nn.Linear(64, 64), torch.nn.ELU(),
                                         torch.nn.Linear(64, out)).to(dev)
    return pack_actor_critic(mk(2), mk(1), torch.tensor([0.7, 1.3], device=dev), 14, dev)


def _buffers(ops, sims, acts):
    f32 = lambda *s: torch.empty(s, dtype=torch.float32, device=DEV)
    u8 = lambda *s: torch.empty(s, dtype=torch.uint8, device=DEV)
    bufs = []
    for op, s, t in ops:
        n = sims[s].num_envs
        b = {}
        if op in ("step", "act", "staged"):
            b = {"obs": f32(n, 14), "rew": f32(n), "term": u8(n), "trunc": u8(n), "log": torch.zeros(16, device=DEV)}
            b["act"] = f32(n, 2) if op == "act" else acts[s][t]
        if op == "act":
            b.update(mean=f32(n, 2), lp=f32(n), val=f32(n))
        if op == "staged":
            b.update(bits=u8(n))
        if op == "rollout":
            from wheeledlab_b200.distributed import RolloutSlab
            b = {"slab": RolloutSlab(ROLL_K, n, 14, 2, DEV), "log": torch.zeros((ROLL_K, 16), device=DEV)}
        if op == "observe":
            b = {"obs": f32(n, 14)}
        bufs.append(b)
    return bufs


def _run_chained(graph):
    """The script on the default kernel (the duo step, chained wherever the previous launch is another set's duo step), one
    stream, no host sync until the end."""
    import wheeledlab_b200 as wl
    from wheeledlab_b200.policy import act_step
    sims = [wl.WheeledSim(_spec(n, 40 + i), DEV) for i, n in enumerate(SIZES)]
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
        obs_in = None                                         # (every act op follows an observe op of its set)
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
            elif op == "rollout":
                sim.rollout(ROLL_K, t, b["slab"], b["log"])
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
            sim.set_step_counter(0)                           # (capture moved the host mirrors only)
        g.replay()
    else:
        body()
    for sim in sims:
        sim.flush_log()
    torch.cuda.synchronize()
    rec = {f"state{i}": s.groups.cpu().numpy() for i, s in enumerate(sims)}
    rec["chained"] = np.array([s.chained_step_count for s in sims])
    rec.update({f"weights{i}": s.rew_weight.cpu().numpy() for i, s in enumerate(sims)})
    for k, b in enumerate(bufs):
        if "slab" in b:
            sl = b["slab"]
            for f, x in (("act", sl.actions), ("obs", sl.obs), ("rew", sl.rewards), ("term", sl.terminated), ("trunc", sl.truncated), ("log", b["log"])):
                rec[f"{k}_{f}"] = x.cpu().numpy()
            continue
        for f, x in b.items():
            if f not in ("mean", "lp", "val", "bits"):
                rec[f"{k}_{f}"] = x.cpu().numpy()
    return rec


def _check_against_thread_per_env(rec, what, graph):
    """Replay the script on thread-per-env sims, one op at a time, with the actions the chained run used (these stand in for
    the oracle: test_gpu_parity.py and test_duo_coverage_gpu.py hold the thread-per-env kernel to it bit for bit).  Also
    check that the chained run launched exactly the chained steps the sequence allows."""
    import wheeledlab_b200 as wl
    sims = [wl.WheeledSim(_spec(n, 40 + i), DEV) for i, n in enumerate(SIZES)]
    w0 = []
    for s in sims:
        s.set_kernel_variant(1); s.startup(); s.reset(None, 0); w0.append(s.rew_weight.cpu().numpy())
    ops, _ = _script(graph)
    exp = _expected_chained(ops)
    assert exp > 100 and int(rec["chained"].sum()) == exp, f"{what}: {rec['chained'].tolist()} chained steps, expected {exp} in all"
    n_done = 0
    for k, (op, s, t) in enumerate(ops):
        sim, where = sims[s], f"{what}: {op} #{k} of set {s} ({SIZES[s]} envs) at t={t}"
        if op == "rollout":
            for j in range(ROLL_K):
                log = torch.zeros(16, device=DEV)
                obs, rew, term, trunc = sim.step(torch.from_numpy(rec[f"{k}_act"][j]).to(DEV), t + j, log=log)
                sim.flush_log()
                for name, a, b in (("obs", obs, "obs"), ("rew", rew, "rew"), ("term", term, "term"), ("trunc", trunc, "trunc")):
                    a = a.cpu().numpy()
                    assert np.array_equal(a.view(np.uint8), rec[f"{k}_{b}"][j].view(np.uint8)), f"{where}+{j}: {name} differs"
                lg, got = log.cpu().numpy(), rec[f"{k}_log"][j]
                assert np.allclose(got[:8], lg[:8], rtol=1e-5, atol=1e-4) and np.array_equal(got[8:11], lg[8:11]), f"{where}+{j}: log differs"
                n_done += int((term | trunc).sum().item())
        elif op == "reset":
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
            n_done += int((term | trunc).sum().item())
    for i, s in enumerate(sims):
        assert np.array_equal(_bits(rec[f"state{i}"]), _bits(s.groups.cpu().numpy())), f"{what}: final state of set {i} differs"
        w = s.rew_weight.cpu().numpy()
        assert np.array_equal(_bits(rec[f"weights{i}"]), _bits(w)), f"{what}: reward weights of set {i} differ"
        assert not np.array_equal(w, w0[i]), f"{what}: the curriculum boundary did not move the weights of set {i}"
    assert n_done > 0, "no auto-reset in the sequence"


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["eager", "graph"])
def test_round_robin_env_sets_match_thread_per_env(mode):
    _need_gpu()
    _check_against_thread_per_env(_run_chained(mode == "graph"), mode, mode == "graph")


@pytest.mark.gpu
def test_round_robin_with_pdl_everywhere(tmp_path):
    """The same sequences with WL_PDL=1: the act-step kernel between two duo steps is PDL-launched too and triggers at
    entry, so the duo step after it must not run chained.  The flag is read when the library loads: a child process runs
    the chained side."""
    _need_gpu()
    env = dict(os.environ, WL_PDL="1")
    r = subprocess.run([sys.executable, str(Path(__file__).resolve()), str(tmp_path)], env=env, capture_output=True, text=True,
                       timeout=900, cwd=str(ROOT))
    assert r.returncode == 0, r.stderr[-3000:]
    for mode in ("eager", "graph"):
        with np.load(tmp_path / f"{mode}.npz") as z:
            _check_against_thread_per_env({k: z[k] for k in z.files}, f"WL_PDL=1 {mode}", mode == "graph")


@pytest.mark.gpu
def test_outputs_are_final_for_a_torch_kernel_after_the_next_set():
    """A 4096-env step, then an 8-env step (chained: it may start before the large one has finished), then torch copies of
    the large step's outputs, queued at once: the copies must hold that step's final rows.  The output buffers are reused
    every step, so a copy that ran early would hold the previous step's rows."""
    _need_gpu()
    import wheeledlab_b200 as wl
    big, small = wl.WheeledSim(_spec(4096, 51), DEV), wl.WheeledSim(_spec(8, 52), DEV)
    ref = wl.WheeledSim(_spec(4096, 51), DEV)
    ref.set_kernel_variant(1)
    for s in (big, small, ref):
        s.startup(); s.reset(None, 0)
    K = 40
    acts = torch.stack([big.synth_actions(t) for t in range(K)])
    acts_small = torch.stack([small.synth_actions(t) for t in range(K)])     # (made up front: a launch between the two steps
                                                                             # would start only once the large step was over)
    out = (torch.empty((4096, 14), device=DEV), torch.empty(4096, device=DEV), torch.empty(4096, dtype=torch.uint8, device=DEV),
           torch.empty(4096, dtype=torch.uint8, device=DEV))
    copies = []
    for t in range(K):
        big.step(acts[t], t, out=out)
        small.step(acts_small[t], t)
        copies.append(tuple(x.clone() for x in out))
    torch.cuda.synchronize()
    for t in range(K):
        r = ref.step(acts[t], t)
        for name, a, b in zip(("obs", "rew", "terminated", "truncated"), r, copies[t]):
            assert torch.equal(a, b), f"step {t}: the copy of {name} is not the step's final output"


if __name__ == "__main__":
    dst = Path(sys.argv[1])
    for m in ("eager", "graph"):
        np.savez(dst / f"{m}.npz", **_run_chained(m == "graph"))
