#!/usr/bin/env python
"""N-sweep of the fused step kernel: per-launch duration (CUDA events) and achieved algorithmic HBM GB/s.

    python tools/sweep.py [--sizes 4096,65536,...] [--steps 30] [--task drift]
Prints one JSON object.
"""
import argparse, json, statistics, sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import torch  # noqa: E402
import wheeledlab_b200 as wl  # noqa: E402
from bench import BYTES_PER_ENV_STEP, _peaks  # noqa: E402


TASK = "drift"
VARIANT = 0
BYTES = {"drift": BYTES_PER_ENV_STEP, "hound_4wd": BYTES_PER_ENV_STEP, "elevation": (15 * 16 + 8) + (11 * 16 + 689 * 4 + 4 + 2),
         "visual_cam": BYTES_PER_ENV_STEP - 14 * 4 + 3208 * 4 + 32,    # step state r/w + obs row written (camera 3200 + 8) + pose re-read
         "camera": 3200 * 4 + 32}                                      # wl_camera_kernel alone: 12.8 KB written + pose (pos, quat) read


def one(n, steps, warm, flush):
    spec = {"drift": lambda: wl.drift_task(num_envs=n, seed=42), "hound_4wd": lambda: wl.make_task("hound_4wd", num_envs=n, seed=42), "elevation": lambda: wl.elevation_task(num_envs=n, seed=42),
            "visual_cam": lambda: wl.visual_task(num_envs=n, seed=42, camera="aug"),
            "camera": lambda: wl.visual_task(num_envs=n, seed=42, camera="aug")}[TASK]()
    sim = wl.WheeledSim(spec, "cuda:0")
    if VARIANT:
        sim.set_kernel_variant(VARIANT)
    sim.startup(); sim.reset(None, 0)
    acts = [sim.synth_actions(t) for t in range(4)]
    outs = tuple(torch.empty_like(x) for x in sim.step(acts[0], 0))
    for t in range(1, warm + 1):
        sim.step(acts[t % 4], t, out=outs)
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(steps)]
    torch.cuda.synchronize()
    for k in range(steps):
        if flush is not None:
            flush.fill_(0.0)
        if TASK == "camera":                             # the camera kernel alone (state left by the warm-up steps)
            ev[k][0].record(); sim.camera(warm + 1 + k, outs[0]); ev[k][1].record()
        else:
            ev[k][0].record(); sim.step(acts[k % 4], warm + 1 + k, out=outs); ev[k][1].record()
    torch.cuda.synchronize()
    ms = [a.elapsed_time(b) for a, b in ev]
    med = statistics.median(ms)
    return {"envs": n, "kernel_us_median": med * 1e3, "kernel_us_min": min(ms) * 1e3,
            "env_steps_per_s": n / (med * 1e-3), "achieved_GBps": BYTES[TASK] * n / (med * 1e-3) / 1e9}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="1024,4096,16384,65536,262144,1048576,4194304")
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warm", type=int, default=5)
    ap.add_argument("--no-flush", action="store_true")
    ap.add_argument("--task", default="drift", choices=["drift", "hound_4wd", "elevation", "visual_cam", "camera"])
    ap.add_argument("--variant", type=int, default=0, help="0 auto, 1 thread/env, 4 quad/env")
    a = ap.parse_args()
    global TASK, VARIANT
    TASK = a.task
    VARIANT = a.variant
    peak, src = _peaks()
    flush = None if a.no_flush else torch.empty(256 * 1024 * 1024 // 4, dtype=torch.float32, device="cuda:0")
    rows = []
    for n in [int(x) for x in a.sizes.split(",")]:
        r = one(n, a.steps, a.warm, flush)
        r["frac_of_peak"] = r["achieved_GBps"] / peak
        rows.append(r)
        print(json.dumps(r), file=sys.stderr, flush=True)
    kname = {"camera": "wl_camera_kernel", "visual_cam": "wl_step[_quad]_kernel<visual> + wl_camera_kernel"}.get(
        TASK, f"wl_step[_quad]_kernel<{TASK}>" + (" + wl_scan_kernel<TMA>" if TASK == "elevation" else ""))
    print(json.dumps({"kernel": kname,
                      "bytes_per_env_step": BYTES[TASK], "peak_GBps": peak,
                      "peak_source": src, "l2_flush_between_launches": not a.no_flush, "rows": rows}))


if __name__ == "__main__":
    main()
