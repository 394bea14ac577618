#!/usr/bin/env python
"""Kernel A/B experiments with the bench protocol (L2 flushed between steps, CUDA events around each step launch).

    python tools/kexp.py build                 # here (nvcc cross-compiles): build_ab/libwl_<name>.so for every variant
    python tools/kexp.py run [--envs 4096]     # on the GPU: one subprocess per variant, one JSON line each
Variants are sets of -D macros of csrc/wl_api.cu (experiment switches, never part of the shipped library)."""
import json
import os
import statistics
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
AB = ROOT / "build_ab"
VARIANTS = json.loads(os.environ.get("KEXP_VARIANTS", "null")) or {
    "base": [],
}


def build():
    sys.path.insert(0, str(ROOT))
    import importlib.util
    spec = importlib.util.spec_from_file_location("_wl_build", ROOT / "wheeledlab_b200" / "build.py")
    b = importlib.util.module_from_spec(spec); spec.loader.exec_module(b)
    AB.mkdir(exist_ok=True)
    procs = []
    for name, macros in VARIANTS.items():
        out = AB / f"libwl_{name}.so"
        cmd = [b.NVCC, *b.NVCC_FLAGS, *[f"-D{m}" for m in macros], "-o", str(out), str(b.CSRC / "wl_api.cu")]
        procs.append((name, subprocess.Popen(cmd, cwd=str(ROOT))))
    for name, p in procs:
        assert p.wait() == 0, name
    print("built", list(VARIANTS))


def child(envs, steps, warm, task):
    sys.path.insert(0, str(ROOT))
    import torch
    import wheeledlab_b200 as wl
    from wheeledlab_b200.sim import _stream_ptr
    dev = "cuda:0"
    spec = wl.make_task(task, num_envs=envs, seed=42)
    sim = wl.WheeledSim(spec, dev); sim.startup(); sim.reset(None, 0)
    KV = int(os.environ.get("KEXP_KVARIANT", "0"))
    sim.set_kernel_variant(KV)
    K, W = steps, warm
    acts = torch.stack([sim.synth_actions(t) for t in range(W + K)])
    out = (torch.empty((envs, sim.obs_dim), device=dev), torch.empty(envs, device=dev), torch.empty(envs, dtype=torch.uint8, device=dev),
           torch.empty(envs, dtype=torch.uint8, device=dev))
    log = torch.empty(16, device=dev)
    flush = torch.empty(256 * 1024 * 1024 // 4, dtype=torch.float32, device=dev)
    t = 0
    for _ in range(W):
        sim.step(acts[t], t, out=out, log=log); flush.fill_(0.0); t += 1
    torch.cuda.synchronize()
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(K)]
    for k in range(K):
        ev[k][0].record(); sim.step(acts[t], t, out=out, log=log); ev[k][1].record(); flush.fill_(0.0); t += 1
    torch.cuda.synchronize()
    cold = [a.elapsed_time(b) * 1e3 for a, b in ev]
    # warm: graph of K steps
    g = torch.cuda.CUDAGraph(); s = torch.cuda.Stream(); s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        with torch.cuda.graph(g, stream=s):
            for k in range(K):
                sim.step(acts[W + k], t + k, out=out, log=log)
    torch.cuda.current_stream().wait_stream(s)
    g.replay(); torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(); g.replay(); e1.record(); torch.cuda.synchronize()
    warm_us = e0.elapsed_time(e1) * 1e3 / K
    # working set larger than L2 instead of a flush kernel: M independent env sets stepped round-robin, back to back
    M = int(os.environ.get("KEXP_SETS", "160"))
    sims = []
    for m in range(M):
        sm = wl.WheeledSim(wl.make_task(task, num_envs=envs, seed=42 + m), dev); sm.startup(); sm.reset(None, 0); sm.set_kernel_variant(KV); sims.append(sm)
    outs = [tuple(torch.empty_like(x) for x in out) for _ in range(M)]
    bound = [sims[m].bind_step(acts[m % (W + K)], outs[m]) for m in range(M)]
    tt = [0] * M
    def rot(nsteps, k0):
        for k in range(nsteps):
            m = (k0 + k) % M
            bound[m](tt[m]); tt[m] += 1
    rot(2 * M, 0); torch.cuda.synchronize()
    RK = 4 * M
    r0, r1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    r0.record(); rot(RK, 0); r1.record(); torch.cuda.synchronize()
    rot_us = r0.elapsed_time(r1) * 1e3 / RK
    # launch floors: graphs of 200 empty kernels (no parameter / the 1.5 KB wl_config parameter), and stream launches of the same
    floors = {}
    geo = ((envs * 4 + 31) // 32 + 1, 32)
    for name, fn in (("null", lambda: wl.lib.wl_test_null(geo[0], geo[1], _stream_ptr(sim.device))),
                     ("null_cfg", lambda: wl.lib.wl_test_null_cfg(sim._h, geo[0], geo[1], _stream_ptr(sim.device)))):
        gg = torch.cuda.CUDAGraph(); ss = torch.cuda.Stream(); ss.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(ss):
            with torch.cuda.graph(gg, stream=ss):
                for _ in range(200):
                    fn()
        torch.cuda.current_stream().wait_stream(ss)
        gg.replay(); torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); gg.replay(); b.record(); torch.cuda.synchronize()
        floors[name + "_graph_us"] = a.elapsed_time(b) * 1e3 / 200
        for _ in range(50):
            fn()
        torch.cuda.synchronize()
        a.record()
        for _ in range(400):
            fn()
        b.record(); torch.cuda.synchronize()
        floors[name + "_stream_us"] = a.elapsed_time(b) * 1e3 / 400
    # floor of the protocol: empty kernel of the same geometry between the same events / flushes
    nul = []
    for geo in ((envs * 4 + 31) // 32, 32), ((envs * 4 + 127) // 128, 128):
        evn = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(50)]
        for a, b in evn:
            a.record(); wl.lib.wl_test_null(geo[0], geo[1], _stream_ptr(sim.device)); b.record(); flush.fill_(0.0)
        torch.cuda.synchronize()
        nul.append(statistics.median(a.elapsed_time(b) * 1e3 for a, b in evn))
    print(json.dumps({"variant": os.environ.get("KEXP_NAME"), "task": task, "envs": envs, "cold_us_mean": statistics.mean(cold),
                      "cold_us_median": statistics.median(cold), "cold_us_min": min(cold), "warm_graph_us": warm_us,
                      "rotate_us": rot_us, "floors": floors, "kernel_variant": KV, "rotate_sets": M, "pdl": os.environ.get("WL_PDL", "1"),
                      "null_us_bs32": nul[0], "null_us_bs128": nul[1]}), flush=True)


def run(envs, task):
    for name in VARIANTS:
        for pdl in os.environ.get("KEXP_PDL", "0").split(","):
            for kv in os.environ.get("KEXP_KVARIANTS", "0").split(","):
                env = dict(os.environ, WHEELEDLAB_B200_LIB=str(AB / f"libwl_{name}.so"), KEXP_NAME=name, WL_PDL=pdl, KEXP_KVARIANT=kv)
                subprocess.run([sys.executable, __file__, "child", str(envs), task], env=env, check=False)


if __name__ == "__main__":
    cmd = sys.argv[1] if len(sys.argv) > 1 else "build"
    if cmd == "build":
        build()
    elif cmd == "child":
        child(int(sys.argv[2]), 200, 20, sys.argv[3])
    else:
        envs = int(sys.argv[sys.argv.index("--envs") + 1]) if "--envs" in sys.argv else 4096
        task = sys.argv[sys.argv.index("--task") + 1] if "--task" in sys.argv else "drift"
        run(envs, task)
