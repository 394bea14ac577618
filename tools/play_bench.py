"""Per-step device time of playing a policy: the deterministic rollout (FusedPolicyRollout(deterministic=True)) against the
training rollout at the same size and a torch actor in the same graph form, plus the reference-shaped eager loop and
wl_actor_mean alone.

Workloads: Drift at 1024 and 4096 envs (ELU, T x wl_act_infer_step), Elevation at 1024 and 4096 (ReLU, T x (wl_actor_mean
-> wl_step)), camera Visual at 512 (ReLU, obs_dim 3208).  1024 and 512 are the reference's run-config sizes.  Forms, each
one CUDA graph of T = 200 steps, timed with CUDA events over replays after warm-up and alternated `--runs` times in one
process:
  det    the deterministic rollout
  train  the training FusedPolicyRollout (critic, noise, log-prob)
  torch  a torch actor (cuBLAS addmm + activation) -> wl_step
  eager  play_policy.py's loop, actions = policy(obs); env.step(actions) per step, with the torch actor, on a host clock
         that ends in a synchronise
wl_actor_mean alone is timed at obs_dim 689 (4096 rows), with its FP32 share from 2 (689 64 + 64 64 + 64 2) FLOPs per row.
The card's name and power limit are read in the same call.

    python tools/play_bench.py --out results/h100/playback
"""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))

WORKLOADS = [("drift", 1024), ("drift", 4096), ("elevation", 1024), ("elevation", 4096), ("visual", 512)]
FP32_PEAK = 67e12                      # H100 SXM data sheet, dense FP32


def _timed(fn, reps):
    fn(); torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / reps            # us per call


def workload(task, n, T, seed=0):
    import wheeledlab_b200 as wl
    from wheeledlab_b200.policy import ACTIVATIONS, FusedPolicyRollout, _blob_layers, pack_actor_critic
    from wheeledlab_b200.runs import task_activation
    dev = "cuda:0"
    ids = {"drift": "Isaac-MushrDriftRL-v0", "elevation": "Isaac-MushrElevationRL-v0", "visual": "Isaac-MushrVisualRL-v0"}
    act = task_activation(task)

    def make_env(s):
        return wl.make(ids[task], device=dev, num_envs=n, seed=s)

    envs = [make_env(seed + k) for k in range(4)]
    for e in envs:
        e.reset()
    D = envs[0].sim.obs_dim
    torch.manual_seed(seed)
    A = torch.nn.ELU if act == "elu" else torch.nn.ReLU
    mk = lambda out: torch.nn.Sequential(torch.nn.Linear(D, 64), A(), torch.nn.Linear(64, 64), A(), torch.nn.Linear(64, out))
    blob = pack_actor_critic(mk(2), mk(1), torch.ones(2), D, dev)
    actor, _, _ = _blob_layers(blob, D)
    f = ACTIVATIONS[act]

    def torch_actor(x):
        for k, (w, b) in enumerate(actor):
            x = torch.addmm(b, x, w)
            if k < 2:
                x = f(x)
        return x

    det = FusedPolicyRollout(envs[0].sim, blob, T, activation=act, deterministic=True).capture(0)
    train = FusedPolicyRollout(envs[1].sim, blob, T, activation=act).capture(0)
    sim_t = envs[2].sim
    slab_t = FusedPolicyRollout(sim_t, blob, T, activation=act, deterministic=True).slab

    def torch_body():
        for k in range(T):
            slab_t.actions[k].copy_(torch_actor(slab_t.obs_in[k]))
            sim_t.step(slab_t.actions[k], wl.WheeledSim.device_counter_plus(k), out=slab_t.step_outputs(k))
        sim_t.advance_counter(T)
        slab_t.obs_in[0].copy_(slab_t.obs[T - 1])

    sim_t.observe(0, 0, out=slab_t.obs_in[0]); sim_t.set_step_counter(0)
    st = torch.cuda.Stream(); st.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(st):
        torch_actor(slab_t.obs_in[0])                                        # cuBLAS warm-up outside the capture
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=st):
            torch_body()
    torch.cuda.current_stream().wait_stream(st)
    sim_t.set_step_counter(0)
    base = [0]

    def torch_rep():
        g.replay(); base[0] += T; sim_t.note_device_counter(base[0])

    env_e = envs[3]

    def eager():
        obs, _ = env_e.get_observations()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        with torch.inference_mode():
            for _ in range(T):
                actions = torch_actor(obs)
                obs_d, _, _, _, _ = env_e.step(actions)
                obs = obs_d["policy"]
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1e6 / T

    forms = {"det": lambda: _timed(det.run, 5) / T, "train": lambda: _timed(train.run, 5) / T, "torch": lambda: _timed(torch_rep, 5) / T,
             "eager": eager}
    return D, act, forms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200, help="T steps per graph")
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("play_bench needs a CUDA device")
    from wheeledlab_b200.policy import actor_mean, pack_actor_critic
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()[0]
    out = Path(a.out) if a.out else None
    if out:
        out.mkdir(parents=True, exist_ok=True)
        (out / "gpu.csv").write_text("name, power.limit [W], clocks.max.sm [MHz]\n" + gpu + "\n")
    lines = []
    for task, n in WORKLOADS:
        D, act, forms = workload(task, n, a.steps)
        for r in range(a.runs):
            res = {"run": r + 1, "gpu": gpu, "task": task, "envs": n, "obs_dim": D, "activation": act, "T": a.steps}
            for name, fn in forms.items():
                res[f"{name}_us_per_step"] = fn()
            print(json.dumps(res), flush=True)
            lines.append(json.dumps(res))
        torch.cuda.empty_cache()
    # wl_actor_mean alone at the Elevation width
    D, n = 689, 4096
    torch.manual_seed(0)
    mk = lambda out: torch.nn.Sequential(torch.nn.Linear(D, 64), torch.nn.ReLU(), torch.nn.Linear(64, 64), torch.nn.ReLU(), torch.nn.Linear(64, out))
    blob = pack_actor_critic(mk(2), mk(1), torch.ones(2), D, "cuda:0")
    obs = torch.randn(n, D, device="cuda:0")
    mean = torch.empty(n, 2, device="cuda:0")
    flop = 2 * n * (D * 64 + 64 * 64 + 64 * 2)
    calls = 50                                         # one graph of 50 launches: device time, not the Python call
    g = torch.cuda.CUDAGraph()
    st = torch.cuda.Stream(); st.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(st):
        actor_mean(blob, D, obs, "relu", out=mean)
        with torch.cuda.graph(g, stream=st):
            for _ in range(calls):
                actor_mean(blob, D, obs, "relu", out=mean)
    torch.cuda.current_stream().wait_stream(st)
    for r in range(a.runs):
        us = _timed(g.replay, 10) / calls
        res = {"run": r + 1, "gpu": gpu, "kernel": "wl_actor_mean", "rows": n, "obs_dim": D, "activation": "relu", "us": us,
               "gflop": flop / 1e9, "share_of_fp32_peak": flop / (us * 1e-6) / FP32_PEAK}
        print(json.dumps(res), flush=True)
        lines.append(json.dumps(res))
    if out:
        (out / "play_bench.jsonl").write_text("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
