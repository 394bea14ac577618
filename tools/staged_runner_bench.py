"""What training with host-side Python terms costs: whole FusedOnPolicyRunner iterations, Drift 4096 envs x 128 steps with
PPOConfig(), host clock between the ends of consecutive iterations (each ends in the read-back's synchronise), three
variants alternated in one process:

    fused     no Python terms: the one-graph iteration
    staged0   one Python reward term of weight 0: the staged rollout's machinery alone (policy, stage a, stage b, the
              per-step log entries; the term itself is skipped)
    staged    one reference-style reward term (forward speed from scene["robot"].data, weight 1)

and the policy kernels alone at the same size (CUDA events over graph replays of 100 launches on device counters):
wl_policy_act_elu, wl_act_step and wl_step, so that wl_policy_act_elu can be set against wl_act_step minus wl_step.

    python tools/staged_runner_bench.py [--envs 4096] [--steps 128] [--runs 3] [--iters 10] --out results.json
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

WARMUP = 2


def forward_speed(env):
    return env.scene["robot"].data.root_lin_vel_b[:, 0]


def iteration_ms(variant: str, n: int, T: int, iters: int) -> list:
    import wheeledlab_b200 as wl
    from wheeledlab_b200.learner import FusedOnPolicyRunner
    from wheeledlab_b200.runs import agent_cfg
    env = wl.make("Isaac-MushrDriftRL-v0", device="cuda:0", num_envs=n, seed=0)
    if variant != "fused":
        env.add_reward_term("forward_speed", forward_speed, 0.0 if variant == "staged0" else 1.0)
    torch.manual_seed(0)
    runner = FusedOnPolicyRunner(env, agent_cfg("elu", steps=T), device="cuda:0")
    stamps = []
    runner.callback = lambda it, log: stamps.append(time.perf_counter())
    torch.cuda.synchronize()
    runner.learn(WARMUP + iters + 1)
    env.close()
    return [1e3 * (b - a) for a, b in zip(stamps[WARMUP:], stamps[WARMUP + 1:])]


def kernel_us(n: int, launches: int = 100, replays: int = 20) -> dict:
    import wheeledlab_b200 as wl
    from wheeledlab_b200 import WheeledSim
    from wheeledlab_b200.policy import act_step, pack_actor_critic, policy_act
    dev = "cuda:0"
    out = {}
    for name in ("wl_policy_act_elu", "wl_act_step", "wl_step"):
        sim = WheeledSim(wl.drift_task(num_envs=n, seed=0), dev)
        sim.startup(); sim.reset(None, 0)
        D = sim.obs_dim
        torch.manual_seed(0)
        mk = lambda o: torch.nn.Sequential(torch.nn.Linear(D, 64), torch.nn.ELU(), torch.nn.Linear(64, 64), torch.nn.ELU(), torch.nn.Linear(64, o))
        blob = pack_actor_critic(mk(2), mk(1), torch.ones(2), D, dev)
        obs_in = sim.observe(0, 0)
        pol = [torch.empty((n, 2), device=dev), torch.empty((n, 2), device=dev), torch.empty(n, device=dev), torch.empty(n, device=dev)]
        step_out = (torch.empty((n, D), device=dev), torch.empty(n, device=dev), torch.empty(n, dtype=torch.uint8, device=dev),
                    torch.empty(n, dtype=torch.uint8, device=dev))
        act = sim.synth_actions(0)

        def body():
            for k in range(launches):
                t = WheeledSim.device_counter_plus(k)
                if name == "wl_policy_act_elu":
                    policy_act(sim, obs_in, blob, *pol, t, activation="elu")
                elif name == "wl_act_step":
                    act_step(sim, obs_in, blob, *pol, step_out, None, t)
                else:
                    sim.step(act, t, out=step_out)
            sim.advance_counter(launches)

        sim.set_step_counter(0)
        g, s = torch.cuda.CUDAGraph(), torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s), torch.cuda.graph(g, stream=s):
            body()
        torch.cuda.current_stream().wait_stream(s)
        sim.set_step_counter(0)
        base = 0
        g.replay(); base += launches; sim.note_device_counter(base)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(replays):
            g.replay()
        e1.record(); torch.cuda.synchronize()
        base += replays * launches; sim.note_device_counter(base)
        out[name] = e0.elapsed_time(e1) * 1e3 / (replays * launches)
        sim.close()
    out["wl_act_step_minus_wl_step"] = out["wl_act_step"] - out["wl_step"]
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=128)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--iters", type=int, default=10, help="timed iterations per run (after %d warm-up iterations)" % WARMUP)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("staged_runner_bench: no CUDA device (nothing is measured without one)")
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    res = {"gpu": smi, "envs": a.envs, "steps": a.steps, "iters": a.iters, "iteration_ms": {}, "kernel_us": []}
    variants = ("fused", "staged0", "staged")
    for v in variants:
        res["iteration_ms"][v] = []
    for _ in range(a.runs):
        for v in variants:
            res["iteration_ms"][v].append(iteration_ms(v, a.envs, a.steps, a.iters))
    for _ in range(a.runs):
        res["kernel_us"].append(kernel_us(a.envs))
    res["median_iteration_ms"] = {v: statistics.median(x for run in res["iteration_ms"][v] for x in run) for v in variants}
    line = json.dumps(res)
    print(line)
    if a.out:
        Path(a.out).parent.mkdir(parents=True, exist_ok=True)
        Path(a.out).write_text(line + "\n")


if __name__ == "__main__":
    main()
