"""Time one PPO update at the reference's sizes (4096 envs x 128 steps, PPOConfig(): 5 epochs x 4 mini-batches of 131 072):

  fused   wl_ppo_update (learner.FusedPPO) captured in a CUDA graph; CUDA events around graph replays, after warm-up
  torch   the torch restatement of rsl_rl PPO.update() (tests/ppo_reference.py; ReLU: ppo_reference_relu.py), eager with its host syncs; host clock
          around whole updates, each ending in a device synchronise
  iter    one whole training iteration (rollout + bootstrap + GAE + fused update) as one CUDA graph (learner.PPOIteration)

The three variants alternate, `--runs` times, in one process; the card's name and power limit are read in the same call.
``--task elevation`` runs the Elevation network (obs_dim 689, ReLU: wl_ppo_update_wide) on an Elevation rollout.
FLOPs are counted from shapes (forward + weight gradients + input gradients of layers 2 and 3, per sample); the fused
update's FLOP rate over the FP32 data-sheet rate (67 TFLOP/s, H100 SXM) is its kernel share.  One JSON file per run.

    python tools/ppo_update_bench.py --out results/h100/ppo_update
    python tools/ppo_update_bench.py --task elevation --out results/h100/ppo_update_elev
"""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT)); sys.path.insert(0, str(ROOT / "tests"))

FP32_PEAK = 67e12


TASKS = {"drift": ("drift_task", "elu"), "elevation": ("elevation_task", "relu")}


def flops_per_sample(obs_dim: int, hidden: int = 64) -> int:
    fwd = sum(2 * (obs_dim * hidden + hidden * hidden + hidden * out) for out in (2, 1))
    dx = sum(2 * (hidden * hidden + hidden * out) for out in (2, 1))          # layer-1 input gradient is not needed
    return 2 * fwd + dx                                                        # forward + weight gradients + dx


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=128)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--reps", type=int, default=20, help="updates timed per variant and run")
    ap.add_argument("--task", choices=list(TASKS), default="drift")
    ap.add_argument("--out", default=None, help="default: results/h100/ppo_update (drift), results/h100/ppo_update_elev")
    a = ap.parse_args()
    a.out = a.out or ("results/h100/ppo_update" if a.task == "drift" else "results/h100/ppo_update_elev")
    make, activation = TASKS[a.task]
    import wheeledlab_b200 as wl
    from ppo_reference_relu import torch_ppo
    from wheeledlab_b200.learner import FusedPPO, PPOConfig, PPOIteration, compute_returns
    from wheeledlab_b200.policy import FusedPolicyRollout, critic_value, pack_actor_critic
    if not torch.cuda.is_available():
        raise SystemExit("ppo_update_bench needs a CUDA device")
    dev = "cuda:0"
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()[0]
    cfg = PPOConfig()
    torch.manual_seed(0)
    sim = wl.WheeledSim(getattr(wl, make)(num_envs=a.envs, seed=0), dev); sim.startup(); sim.reset(None, 0)
    D = sim.obs_dim
    act = {"elu": torch.nn.ELU, "relu": torch.nn.ReLU}[activation]
    mk = lambda out: torch.nn.Sequential(torch.nn.Linear(D, 64), act(), torch.nn.Linear(64, 64), act(), torch.nn.Linear(64, out))
    blob0 = pack_actor_critic(mk(2), mk(1), torch.ones(2), D, dev)
    roll = FusedPolicyRollout(sim, blob0.clone(), a.steps, activation=activation).capture(0)
    slab = roll.run()
    last = critic_value(roll.blob, D, roll.obs0, activation)
    ret, adv = compute_returns(slab.rewards, slab.values, last, slab.terminated | slab.truncated, cfg.gamma, cfg.lam, time_outs=slab.truncated)
    n = a.envs * a.steps
    perm = torch.randperm(n, device=dev)
    flop = flops_per_sample(D) * n * cfg.num_learning_epochs

    fused = FusedPPO(blob0.clone(), D, cfg, activation)
    fused.update(slab, ret, adv, perm)
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream(); s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s), torch.cuda.graph(g, stream=s):
        fused.update(slab, ret, adv, perm)
    torch.cuda.current_stream().wait_stream(s)

    sim2 = wl.WheeledSim(getattr(wl, make)(num_envs=a.envs, seed=1), dev); sim2.startup(); sim2.reset(None, 0)
    it = PPOIteration(sim2, blob0.clone(), cfg, a.steps, activation=activation).start(0, capture=True)

    def time_fused():
        fused.blob.copy_(blob0)                        # the same starting weights every run
        g.replay(); torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(a.reps):
            g.replay()
        e1.record(); torch.cuda.synchronize()
        return e0.elapsed_time(e1) / a.reps

    def time_torch():
        ts = []
        for k in range(max(2, a.reps // 5) + 1):
            ref = torch_ppo(blob0, D, cfg, torch.float32, activation)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            ref.update(slab.obs_in, slab.actions, slab.values, slab.log_prob, slab.mean, ret, adv, perm)
            torch.cuda.synchronize()
            if k:                                      # the first is warm-up
                ts.append((time.perf_counter() - t0) * 1e3)
        return sum(ts) / len(ts)

    def time_iter():
        it.run(perm); torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(a.reps):
            it.run(perm)
        e1.record(); torch.cuda.synchronize()
        return e0.elapsed_time(e1) / a.reps

    out = Path(a.out); out.mkdir(parents=True, exist_ok=True)
    for r in range(a.runs):
        res = {"run": r + 1, "gpu": gpu, "task": a.task, "obs_dim": D, "envs": a.envs, "steps": a.steps, "epochs": cfg.num_learning_epochs,
               "mini_batches": cfg.num_mini_batches, "mini_batch": n // cfg.num_mini_batches, "reps": a.reps}
        res["fused_update_ms"] = time_fused()
        res["torch_update_ms"] = time_torch()
        res["iteration_ms"] = time_iter()
        res["update_gflop"] = flop / 1e9
        res["fused_tflops"] = flop / (res["fused_update_ms"] * 1e-3) / 1e12
        res["fused_kernel_share_of_fp32_peak"] = res["fused_tflops"] * 1e12 / FP32_PEAK
        res["torch_tflops"] = flop / (res["torch_update_ms"] * 1e-3) / 1e12
        res["speedup_vs_torch"] = res["torch_update_ms"] / res["fused_update_ms"]
        print(json.dumps(res), flush=True)
        (out / f"bench_run{r + 1}.json").write_text(json.dumps(res) + "\n")


if __name__ == "__main__":
    main()
