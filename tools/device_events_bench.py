"""What device event terms cost (DESIGN 6p), one GPU:

    elevation  whole FusedOnPolicyRunner iterations on Elevation (--envs x --steps, host clock between the ends of
               consecutive iterations): "python", IsaacLab's push as a host-side Python interval event (the staged
               iteration), against "device", the same push as a device event term (one graph), and "none", the env without
               the push (the fused iteration), alternated over --runs rounds
    drift      the same on Drift: "none", the fused baseline iteration, against "device", one device push added
    kernel     wl_device_events alone at 4096 and 8192 envs with 1 and 8 terms, CUDA events over graph replays of 100 launches

    python tools/device_events_bench.py [--envs 4096] [--steps 128] [--runs 3] [--iters 10] --out results.json
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

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "shims"))

DEV = "cuda:0"
WARMUP = 2
PUSH = {"x": (-0.5, 0.5), "y": (-0.5, 0.5), "yaw": (-0.5, 0.5)}
INTERVAL = (1.0, 3.0)


def python_push(env, env_ids, velocity_range):
    """push_by_setting_velocity restated in torch, as a user would write it for a host-side event term."""
    robot = env.scene["robot"]
    vel = torch.cat([robot.data.root_lin_vel_w[env_ids], robot.data.root_ang_vel_w[env_ids]], dim=1)
    for j, c in enumerate(("x", "y", "z", "roll", "pitch", "yaw")):
        lo, hi = velocity_range.get(c, (0.0, 0.0))
        vel[:, j] += torch.rand(len(env_ids), device=vel.device) * (hi - lo) + lo
    robot.write_root_velocity_to_sim(vel, env_ids=env_ids)


def iteration_ms(task: str, variant: str, n: int, T: int, iters: int) -> list:
    import wheeledlab_b200 as wl
    from isaaclab.envs import mdp
    from wheeledlab_b200.env import ManagerBasedRLEnv
    from wheeledlab_b200.learner import FusedOnPolicyRunner
    from wheeledlab_b200.runs import agent_cfg
    spec = wl.elevation_task(num_envs=n, seed=0) if task == "elevation" else wl.drift_task(num_envs=n, seed=0)
    env = ManagerBasedRLEnv(spec, device=DEV)
    if variant == "python":
        env.add_event_term("push", python_push, "interval", {"velocity_range": PUSH}, interval_range_s=INTERVAL)
    elif variant == "device":
        env.add_device_event_term("push", mdp.push_by_setting_velocity, "interval", INTERVAL, {"velocity_range": PUSH})
    torch.manual_seed(0)
    runner = FusedOnPolicyRunner(env, agent_cfg("relu" if task == "elevation" else "elu", steps=T), device=DEV)
    stamps = []
    runner.callback = lambda it, log: stamps.append(time.perf_counter())
    torch.cuda.synchronize()
    runner.learn(WARMUP + iters + 1)
    env.close()
    return [1e3 * (b - a) for a, b in zip(stamps[WARMUP:], stamps[WARMUP + 1:])]


def kernel_us(n: int, terms: int, launches: int = 100, replays: int = 20) -> float:
    import wheeledlab_b200 as wl
    sim = wl.WheeledSim(wl.elevation_task(num_envs=n, seed=0), DEV)
    ranges = [PUSH.get(c, (0.0, 0.0)) for c in ("x", "y", "z", "roll", "pitch", "yaw")]
    sim.set_device_events([("interval", INTERVAL, ranges)] * terms)
    sim.startup(); sim.reset(None, 0)
    term = (torch.rand(n, device=DEV) < 0.01).to(torch.uint8)
    trunc = torch.zeros(n, dtype=torch.uint8, device=DEV)
    g, s = torch.cuda.CUDAGraph(), torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s), torch.cuda.graph(g, stream=s):
        for k in range(launches):
            sim.device_events(term, trunc, k)
    torch.cuda.current_stream().wait_stream(s)
    g.replay(); torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(replays):
        g.replay()
    e1.record(); torch.cuda.synchronize()
    sim.close()
    return e0.elapsed_time(e1) * 1e3 / (replays * launches)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=128)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--iters", type=int, default=10, help="timed iterations per run (after %d warm-up iterations)" % WARMUP)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("device_events_bench: no CUDA device (nothing is measured without one)")
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    res = {"gpu": smi, "envs": a.envs, "steps": a.steps, "iters": a.iters,
           "iteration_ms": {"elevation/python": [], "elevation/device": [], "elevation/none": [], "drift/none": [], "drift/device": []}, "kernel_us": {}}
    for _ in range(a.runs):
        for key in res["iteration_ms"]:
            task, variant = key.split("/")
            res["iteration_ms"][key].append(statistics.median(iteration_ms(task, variant, a.envs, a.steps, a.iters)))
    for n in (4096, 8192):
        for k in (1, 8):
            res["kernel_us"][f"{n}x{k}"] = kernel_us(n, k)
    res["summary"] = {"iteration_ms": {k: statistics.median(v) for k, v in res["iteration_ms"].items()}}
    line = json.dumps(res)
    print(line)
    if a.out:
        Path(a.out).parent.mkdir(parents=True, exist_ok=True)
        Path(a.out).write_text(line + "\n")


if __name__ == "__main__":
    main()
