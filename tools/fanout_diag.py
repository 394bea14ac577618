"""Where does the time of the N>1 slab exchange go?  torchrun --nproc-per-node N tools/fanout_diag.py
Graphs of T env steps (Drift, 4096 envs/rank) in the exchange forms, each replayed several times (first replay = first touch
of the peer mappings); prints per-replay microseconds, max over ranks.  Diagnostic only."""
import json, os, sys
import torch, torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import wheeledlab_b200 as wl
from wheeledlab_b200.distributed import SymmetricRolloutSlab, RolloutSlab

rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
torch.cuda.set_device(local); dev = torch.device("cuda", local)
dist.init_process_group("nccl", device_id=dev)
E, T, M, REPS = 4096, int(os.environ.get("T", 10)), int(os.environ.get("M", 16)), 6
sims = []
for m in range(M):
    spec = wl.make_task("Isaac-MushrDriftRL-v0", num_envs=E, seed=17 + m, env_id_offset=rank * E)
    s = wl.WheeledSim(spec, dev); s.startup(); s.reset(None, 0); sims.append(s)
sym = SymmetricRolloutSlab(T, E, 14, 2, dev)
loc = RolloutSlab(T, E, 14, 2, dev)
acts = torch.stack([sims[0].synth_actions(t) for t in range(8)])
tc = [0] * M


kk = [0]


def steps(slab, fan):
    for k in range(T):
        m = kk[0] % M; kk[0] += 1; s = sims[m]
        s.set_peer_fanout(fan)
        s.bind_step(acts[k % 8], slab.step_outputs(k))(tc[m]); tc[m] += 1
        s.set_peer_fanout([])


def forms():
    yield "local", lambda: steps(loc, [])
    yield "symm_nofan", lambda: steps(sym.slab, [])
    yield "fanout", lambda: steps(sym.slab, sym.peer_deltas)
    yield "fanout+barrier", lambda: (steps(sym.slab, sym.peer_deltas), sym.barrier())
    yield "barrier", lambda: sym.barrier()
    yield "barrier_x2", lambda: (sym.barrier(), sym.barrier())
    yield "nofan+ce", lambda: (steps(sym.slab, []), sym.gather_ce())
    yield "ce", lambda: sym.gather_ce()
    yield "nofan+nccl", lambda: (steps(loc, []), loc.all_gather())
    yield "nccl", lambda: loc.all_gather()


loc.all_gather(); steps(loc, []); torch.cuda.synchronize(); dist.barrier()
out = {"world": world, "T": T, "envs_per_rank": E, "env_sets": M}
for name, fn in forms():
    g = torch.cuda.CUDAGraph(); cs = torch.cuda.Stream(device=dev); cs.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(cs):
        with torch.cuda.graph(g, stream=cs):
            fn()
    torch.cuda.current_stream().wait_stream(cs)
    if os.environ.get('UPLOAD'):
        wl.upload_graph(g)
    ts = []
    for r in range(REPS):
        torch.cuda.synchronize(); dist.barrier()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda._sleep(200_000); a.record(); g.replay(); b.record(); torch.cuda.synchronize()
        t = torch.tensor([a.elapsed_time(b) * 1e3], device=dev); dist.all_reduce(t, op=dist.ReduceOp.MAX); ts.append(round(float(t), 2))
    out[name] = ts
    if rank == 0:
        print(name, ts, file=sys.stderr, flush=True)
if rank == 0:
    print(json.dumps(out), flush=True)
dist.barrier(); os._exit(0)
