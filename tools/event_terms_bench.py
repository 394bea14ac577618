"""What host-side event terms cost (DESIGN 6o), Drift family, one GPU:

    stage      the staged step's kernels, stage a + stage b against stage a + stage b1 + stage b2 (no Python in between), CUDA
               events around 200 eager steps, the two alternated over --runs rounds
    timers     wl_event_timers alone at 4096 and 8192 envs with 1 and 8 terms, CUDA events over graph replays of 100 launches
    runner     whole FusedOnPolicyRunner iterations (--envs x --steps, host clock between the ends of consecutive iterations):
               "staged0", one Python reward term of weight 0 (the staged rollout without events), against "interval", one
               Python interval event that kicks the fired envs' forward velocity, alternated over --runs rounds

    python tools/event_terms_bench.py [--envs 4096] [--steps 128] [--runs 3] [--iters 10] --out results.json
"""
from __future__ import annotations

import argparse
import json
import statistics
import subprocess
import sys
import time
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))

DEV = "cuda:0"
WARMUP = 2


def stage_us(n: int, cut: bool, steps: int = 200) -> float:
    import wheeledlab_b200 as wl
    sim = wl.WheeledSim(wl.drift_task(num_envs=n, seed=0), DEV)
    sim.startup(); sim.reset(None, 0)
    act = sim.synth_actions(0)
    rew, bits = torch.empty(n, device=DEV), torch.empty(n, dtype=torch.uint8, device=DEV)
    obs = torch.empty((n, sim.obs_dim), device=DEV)
    term, trunc = torch.empty(n, dtype=torch.uint8, device=DEV), torch.empty(n, dtype=torch.uint8, device=DEV)

    def step(t):
        sim.step_stage_a(act, t, rew=rew, term_bits=bits)
        if cut:
            sim.step_stage_b1(bits, t, out=(term, trunc))
            sim.step_stage_b2(t, out=obs)
        else:
            sim.step_stage_b(bits, t, out=(obs, term, trunc))

    for t in range(20):
        step(t)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for t in range(20, 20 + steps):
        step(t)
    e1.record(); torch.cuda.synchronize()
    sim.close()
    return e0.elapsed_time(e1) * 1e3 / steps


def timers_us(n: int, terms: int, launches: int = 100, replays: int = 20) -> float:
    import wheeledlab_b200 as wl
    sim = wl.WheeledSim(wl.drift_task(num_envs=n, seed=0), DEV)
    sim.startup(); sim.reset(None, 0)
    sim.set_event_timers([(0.5, 2.0)] * terms)
    done = (torch.rand(n, device=DEV) < 0.01).to(torch.uint8)
    fired = torch.empty((terms, n), dtype=torch.uint8, device=DEV)
    g, s = torch.cuda.CUDAGraph(), torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s), torch.cuda.graph(g, stream=s):
        for k in range(launches):
            sim.event_timers(done, k, fired)
    torch.cuda.current_stream().wait_stream(s)
    g.replay(); torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(replays):
        g.replay()
    e1.record(); torch.cuda.synchronize()
    sim.close()
    return e0.elapsed_time(e1) * 1e3 / (replays * launches)


def forward_speed(env):
    return env.scene["robot"].data.root_lin_vel_b[:, 0]


def kick(env, env_ids, speed=0.5):
    robot = env.scene["robot"]
    vel = torch.cat([robot.data.root_lin_vel_w[env_ids], robot.data.root_ang_vel_w[env_ids]], dim=1)
    vel[:, 0] += speed
    robot.write_root_velocity_to_sim(vel, env_ids=env_ids)


def iteration_ms(variant: str, n: int, T: int, iters: int) -> list:
    import wheeledlab_b200 as wl
    from wheeledlab_b200.learner import FusedOnPolicyRunner
    from wheeledlab_b200.runs import agent_cfg
    env = wl.make("Isaac-MushrDriftRL-v0", device=DEV, num_envs=n, seed=0)
    if variant == "staged0":
        env.add_reward_term("forward_speed", forward_speed, 0.0)
    else:
        env.add_event_term("kick", kick, "interval", {"speed": 0.5}, interval_range_s=(1.0, 3.0))
    torch.manual_seed(0)
    runner = FusedOnPolicyRunner(env, agent_cfg("elu", steps=T), device=DEV)
    stamps = []
    runner.callback = lambda it, log: stamps.append(time.perf_counter())
    torch.cuda.synchronize()
    runner.learn(WARMUP + iters + 1)
    env.close()
    return [1e3 * (b - a) for a, b in zip(stamps[WARMUP:], stamps[WARMUP + 1:])]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=128)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--iters", type=int, default=10, help="timed iterations per run (after %d warm-up iterations)" % WARMUP)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("event_terms_bench: no CUDA device (nothing is measured without one)")
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    res = {"gpu": smi, "envs": a.envs, "steps": a.steps, "iters": a.iters,
           "stage_us": {"a+b": [], "a+b1+b2": []}, "timers_us": {}, "iteration_ms": {"staged0": [], "interval": []}}
    for _ in range(a.runs):
        res["stage_us"]["a+b"].append(stage_us(a.envs, False))
        res["stage_us"]["a+b1+b2"].append(stage_us(a.envs, True))
    for n in (4096, 8192):
        for k in (1, 8):
            res["timers_us"][f"{n}x{k}"] = timers_us(n, k)
    for _ in range(a.runs):
        for v in ("staged0", "interval"):
            res["iteration_ms"][v].append(statistics.median(iteration_ms(v, a.envs, a.steps, a.iters)))
    res["summary"] = {"stage_us": {k: statistics.median(v) for k, v in res["stage_us"].items()},
                      "iteration_ms": {k: statistics.median(v) for k, v in res["iteration_ms"].items()}}
    line = json.dumps(res)
    print(line)
    if a.out:
        Path(a.out).parent.mkdir(parents=True, exist_ok=True)
        Path(a.out).write_text(line + "\n")


if __name__ == "__main__":
    main()
