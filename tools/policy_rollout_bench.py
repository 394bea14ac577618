"""Per-step time of the Elevation policy rollout (4096 envs, obs_dim 689) as one CUDA graph of T steps, three forms:

  kernel  T x (wl_policy_act -> wl_step): FusedPolicyRollout(activation="relu")
  torch   T x (the same ReLU actor-critic in torch (cuBLAS addmm, relu), a = mean + std * randn -> wl_step), one graph
  step    T x wl_step on a fixed action: the env step alone, for the policy's share

CUDA events around graph replays after warm-up; the forms alternate, `--runs` times, in one process.  The card's name and
power limit are read in the same call.  Layer 1 (4096 x 689 x 128 FMA) sets the FLOP count of the policy.

    python tools/policy_rollout_bench.py --out results/h100/ppo_update_elev
"""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=128, help="T steps per graph")
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--reps", type=int, default=10, help="graph replays timed per form and run")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import wheeledlab_b200 as wl
    from wheeledlab_b200.policy import FusedPolicyRollout, _blob_layers, pack_actor_critic
    if not torch.cuda.is_available():
        raise SystemExit("policy_rollout_bench needs a CUDA device")
    dev, T, n = "cuda:0", a.steps, a.envs
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()[0]
    torch.manual_seed(0)

    def make_sim(seed):
        s = wl.WheeledSim(wl.elevation_task(num_envs=n, seed=seed), dev); s.startup(); s.reset(None, 0)
        return s

    sim = make_sim(0)
    D = sim.obs_dim
    mk = lambda out: torch.nn.Sequential(torch.nn.Linear(D, 64), torch.nn.ReLU(), torch.nn.Linear(64, 64), torch.nn.ReLU(), torch.nn.Linear(64, out))
    blob = pack_actor_critic(mk(2), mk(1), torch.ones(2), D, dev)
    roll = FusedPolicyRollout(sim, blob, T, activation="relu").capture(0)

    # the torch policy in the same graph form: slab rows as FusedPolicyRollout lays them out
    sim_t = make_sim(1)
    slab_t = FusedPolicyRollout(sim_t, blob, T, activation="relu").slab
    actor, critic, std = _blob_layers(blob, D)
    mean_t, val_t = torch.empty(T, n, 2, device=dev), torch.empty(T, n, device=dev)

    def mlp(layers, x):
        for k, (w, b) in enumerate(layers):
            x = torch.addmm(b, x, w)
            if k < 2:
                x = torch.relu(x)
        return x

    def torch_body():
        for k in range(T):
            t = wl.WheeledSim.device_counter_plus(k)
            m = mlp(actor, slab_t.obs_in[k])
            mean_t[k].copy_(m)
            val_t[k].copy_(mlp(critic, slab_t.obs_in[k]).squeeze(-1))
            slab_t.actions[k].copy_(m + std * torch.randn_like(m))
            sim_t.step(slab_t.actions[k], t, out=slab_t.step_outputs(k))
        sim_t.advance_counter(T)
        slab_t.obs_in[0].copy_(slab_t.obs[T - 1])

    sim_s = make_sim(2)
    slab_s = FusedPolicyRollout(sim_s, blob, T, activation="relu").slab
    fixed = torch.full((n, 2), 0.3, device=dev)

    def step_body():
        for k in range(T):
            sim_s.step(fixed, wl.WheeledSim.device_counter_plus(k), out=slab_s.step_outputs(k))
        sim_s.advance_counter(T)

    graphs = {}
    for name, s_, body, slab in (("torch", sim_t, torch_body, slab_t), ("step", sim_s, step_body, slab_s)):
        s_.observe(0, 0, out=slab.obs_in[0]); s_.set_step_counter(0)
        st = torch.cuda.Stream(); st.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(st):
            mlp(actor, slab.obs_in[0]); torch.randn(4, device=dev)                # warm-up outside the capture
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, stream=st):
                body()
        torch.cuda.current_stream().wait_stream(st)
        s_.set_step_counter(0)
        graphs[name] = (g, s_)
    base = {"torch": 0, "step": 0}

    def time_form(name):
        if name == "kernel":
            roll.run(); torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(a.reps):
                roll.run()
            e1.record(); torch.cuda.synchronize()
            return e0.elapsed_time(e1) / (a.reps * T) * 1e3
        g, s_ = graphs[name]

        def rep():
            g.replay(); base[name] += T; s_.note_device_counter(base[name])
        rep(); torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(a.reps):
            rep()
        e1.record(); torch.cuda.synchronize()
        return e0.elapsed_time(e1) / (a.reps * T) * 1e3

    flop = 2 * n * (D * 128 + 64 * 128 + 64 * 3)
    out = Path(a.out) if a.out else None
    if out:
        out.mkdir(parents=True, exist_ok=True)
    for r in range(a.runs):
        res = {"run": r + 1, "gpu": gpu, "task": "elevation", "envs": n, "obs_dim": D, "T": T, "reps": a.reps}
        for name in ("kernel", "torch", "step"):
            res[f"{name}_us_per_step"] = time_form(name)
        res["policy_kernel_us"] = res["kernel_us_per_step"] - res["step_us_per_step"]
        res["policy_torch_us"] = res["torch_us_per_step"] - res["step_us_per_step"]
        res["policy_gflop"] = flop / 1e9
        res["policy_kernel_share_of_fp32_peak"] = flop / (res["policy_kernel_us"] * 1e-6) / 67e12
        print(json.dumps(res), flush=True)
        if out:
            (out / f"policy_rollout_run{r + 1}.json").write_text(json.dumps(res) + "\n")


if __name__ == "__main__":
    main()
