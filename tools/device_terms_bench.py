"""Per-step cost of the device terms: wl_step_terms with 0, 2 and 8 terms against wl_step, Elevation 4096 and Drift 4096,
each as a CUDA graph of 100 steps on device counters, timed with CUDA events; three alternating rounds.  Then whole runner
iterations at Elevation 4096 x 128 (FusedOnPolicyRunner.learn(1), host clock around work that ends in the read-back's
synchronise, between the ends of consecutive iterations): no extra terms, steep_penalty + upright_penalty as device terms,
the same two as Python terms; three alternating rounds of 3 intervals each after one warm-up.  Writes one JSON line per measurement and the GPU's name / power
limit / max SM clock to results/h100/device_terms/ (or --out).

    python tools/device_terms_bench.py [--out DIR] [--reps 20]
"""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

import wheeledlab_b200 as wl                         # noqa: E402
from wheeledlab_b200 import device_terms as dtm      # noqa: E402
from wheeledlab_b200.sim import WheeledSim           # noqa: E402

E, V = dtm.ELEVATION, dtm.VISUAL
TWO = [("steep_penalty", E, dtm.ROLE_REWARD, -1.0, {"thresh_pitch": 0.3}), ("upright_penalty", E, dtm.ROLE_REWARD, -0.01, {"thresh_deg": 10.0})]
EIGHT = TWO + [("forward_vel", E, 0, 1.0, {}), ("forward_wheel_spin", E, 0, 0.01, {}), ("ascending", E, 0, 1.0, {}),
               ("elevation_continuity", E, 0, 1.0, {"threshold_elev": 0.05}), ("low_speed_penalty", V, 0, -0.5, {}),
               ("roll_over", V, dtm.ROLE_TERMINATION, 0.0, {})]


def _table(terms):
    return [(dtm.resolve(n, m).kind, r, w, dtm.param_values(dtm.resolve(n, m), p)) for n, m, r, w, p in terms]


def _graph(sim, variant, K=100):
    n = sim.num_envs
    act = torch.rand((n, 2), device="cuda") * 2 - 1
    out = sim.step(act, 0)
    log, tl = torch.zeros(16, device="cuda"), torch.zeros(8, device="cuda")
    sim.set_step_counter(1)
    s = torch.cuda.Stream(); s.wait_stream(torch.cuda.current_stream())
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s), torch.cuda.graph(g, stream=s):
        for k in range(K):
            c = WheeledSim.device_counter_plus(k)
            if variant == "wl_step":
                sim.step(act, c, out=out, log=log)
            else:
                sim.step_terms(act, c, out=out, log=log, term_log=tl)
        sim.advance_counter(K)
    torch.cuda.current_stream().wait_stream(s)
    return g, (act, out, log, tl)           # the graph's buffers live as long as the graph


def _time(g, reps):
    for _ in range(3):
        g.replay()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        g.replay()
    b.record(); torch.cuda.synchronize()
    return a.elapsed_time(b) * 1000.0 / (reps * 100)


def _py_steep(env, thresh_pitch):
    q = env.sim.root_quat_w
    w, x, y, z = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
    sp = 2.0 * (w * y - z * x)
    pitch = torch.where(sp.abs() >= 1, torch.copysign(torch.full_like(sp, torch.pi / 2), sp), torch.asin(sp)) % (2 * torch.pi)
    return torch.clamp(pitch - thresh_pitch, min=0)


def _py_upright(env, thresh_deg):
    q = env.sim.root_quat_w
    r22 = 1 - 2.0 / (q * q).sum(-1) * (q[:, 1] * q[:, 1] + q[:, 2] * q[:, 2])
    deg = torch.rad2deg(torch.arccos(r22))
    return torch.where(deg > thresh_deg, deg - thresh_deg, 0.0)


def _runners():
    from wheeledlab_b200.env import ManagerBasedRLEnv
    from wheeledlab_b200.learner import FusedOnPolicyRunner
    from wheeledlab_b200.runs import agent_cfg
    out = {}
    for variant in ("fused", "device_terms", "python_terms"):
        env = ManagerBasedRLEnv(wl.elevation_task(num_envs=4096, seed=1))
        if variant == "device_terms":
            env.add_device_reward_term("steep", dtm.resolve("steep_penalty", E), -1.0, {"thresh_pitch": 0.3})
            env.add_device_reward_term("up", dtm.resolve("upright_penalty", E), -0.01, {"thresh_deg": 10.0})
        elif variant == "python_terms":
            env.add_reward_term("steep", _py_steep, -1.0, {"thresh_pitch": 0.3})
            env.add_reward_term("up", _py_upright, -0.01, {"thresh_deg": 10.0})
        torch.manual_seed(0)
        out[variant] = FusedOnPolicyRunner(env, agent_cfg("relu", steps=128), device="cuda:0")
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=str(ROOT / "results" / "h100" / "device_terms"))
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    out = Path(args.out); out.mkdir(parents=True, exist_ok=True)
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv"],
                         capture_output=True, text=True).stdout
    (out / "gpu.csv").write_text(smi)
    graphs = {}
    for task in ("elevation", "drift"):
        for variant, terms in (("wl_step", None), ("terms0", []), ("terms2", TWO), ("terms8", EIGHT)):
            spec = wl.elevation_task(num_envs=4096, seed=1) if task == "elevation" else wl.drift_task(num_envs=4096, seed=1)
            sim = WheeledSim(spec, "cuda:0")
            if terms:
                sim.set_device_terms(_table(terms))
            sim.startup(); sim.reset(None, 0)
            graphs[(task, variant)] = (sim, *_graph(sim, variant))
    with open(out / "bench.jsonl", "w") as f:
        for rnd in range(3):
            for (task, variant), (sim, g, _) in graphs.items():
                us = _time(g, args.reps)
                line = {"round": rnd, "task": task, "num_envs": 4096, "variant": variant, "us_per_step": round(us, 3)}
                print(json.dumps(line)); f.write(json.dumps(line) + "\n")
    del graphs
    import time
    runners = _runners()
    for r in runners.values():
        r.learn(1)                                           # warm-up: capture, first replays
    with open(out / "runner_bench.jsonl", "w") as f:
        for rnd in range(3):
            for variant, r in runners.items():
                ends = []
                r.callback = lambda k, log: ends.append(time.perf_counter())
                r.learn(4)                                   # (each learn captures its graph once: time between iteration ends)
                ms = [(b - a) * 1e3 for a, b in zip(ends, ends[1:])]
                line = {"round": rnd, "task": "elevation", "num_envs": 4096, "T": 128, "variant": variant,
                        "ms_per_iteration": [round(x, 2) for x in ms]}
                print(json.dumps(line)); f.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
