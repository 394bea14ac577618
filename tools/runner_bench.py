"""What the runner's episode statistics cost: wl_episode_stats alone at N x T (CUDA events over graph replays), the whole
Drift iteration graph with and without them (PPOIteration(episode_stats=False / True), alternating runs), and, for
comparison, the same bookkeeping as a torch loop captured in a graph (per t: running sums, the done mask, the masked
record and reset: the form that needs no nonzero() and no host sync, without the last-100 selection).

    python tools/runner_bench.py [--envs 4096] [--steps 128] [--runs 3] --out results.json
"""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))


def graph_time_us(fn, reps_in_graph: int, replays: int) -> float:
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        fn()                                                   # warm-up outside the capture
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s), torch.cuda.graph(g, stream=s):
        for _ in range(reps_in_graph):
            fn()
    torch.cuda.current_stream().wait_stream(s)
    g.replay(); torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(replays):
        g.replay()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / (replays * reps_in_graph)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=128)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--iters", type=int, default=20, help="timed iterations per whole-iteration run")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import wheeledlab_b200 as wl
    from wheeledlab_b200.learner import EpisodeStatistics, PPOConfig, PPOIteration
    from wheeledlab_b200.policy import pack_actor_critic
    dev, N, T = "cuda:0", a.envs, a.steps
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    g = torch.Generator(device=dev).manual_seed(0)
    rew = torch.randn(T, N, device=dev, generator=g)
    term = (torch.rand(T, N, device=dev, generator=g) < 0.004).to(torch.uint8)      # ~ the Drift rollouts' done rate
    trunc = (torch.rand(T, N, device=dev, generator=g) < 0.002).to(torch.uint8)
    ep = EpisodeStatistics(N, T, dev)
    res = {"gpu": smi, "envs": N, "steps": T}
    res["episode_stats_us"] = [graph_time_us(lambda: ep.update(rew, term, trunc), 100, 20) for _ in range(a.runs)]

    cur, ln = torch.zeros(N, device=dev), torch.zeros(N, device=dev)
    rec_r, rec_l = torch.zeros(T, N, device=dev), torch.zeros(T, N, device=dev)
    done = (term | trunc).bool()
    done_f = done.float()

    def torch_loop():
        for t in range(T):
            cur.add_(rew[t]); ln.add_(1.0)
            torch.mul(cur, done_f[t], out=rec_r[t]); torch.mul(ln, done_f[t], out=rec_l[t])
            cur.masked_fill_(done[t], 0.0); ln.masked_fill_(done[t], 0.0)
    res["torch_loop_in_graph_us"] = [graph_time_us(torch_loop, 1, 20) for _ in range(a.runs)]

    def iteration_ms(stats: bool) -> float:
        torch.manual_seed(0)
        sim = wl.WheeledSim(wl.drift_task(num_envs=N, seed=0), dev)
        sim.startup(); sim.reset(None, 0)
        D = sim.obs_dim
        mk = lambda out: torch.nn.Sequential(torch.nn.Linear(D, 64), torch.nn.ELU(), torch.nn.Linear(64, 64), torch.nn.ELU(), torch.nn.Linear(64, out))
        blob = pack_actor_critic(mk(2), mk(1), torch.ones(2), D, dev)
        it = PPOIteration(sim, blob, PPOConfig(), T, episode_stats=stats).start(0)
        perm = torch.randperm(T * N, device=dev)
        for _ in range(3):
            it.run(perm)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(a.iters):
            it.run(perm)
        e1.record(); torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / a.iters
        sim.close()
        return ms

    res["iteration_ms_without"], res["iteration_ms_with"] = [], []
    for _ in range(a.runs):
        res["iteration_ms_without"].append(iteration_ms(False))
        res["iteration_ms_with"].append(iteration_ms(True))
    line = json.dumps(res)
    print(line)
    if a.out:
        Path(a.out).parent.mkdir(parents=True, exist_ok=True)
        Path(a.out).write_text(line + "\n")


if __name__ == "__main__":
    main()
