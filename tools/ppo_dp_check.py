#!/usr/bin/env python
"""torchrun helper for the data-parallel PPO update across GPUs (DESIGN 6j), next to dp_adam_check.py:

1. one wl_ppo_update_dp per rank over torch symmetric memory: the replicas stay bit-identical;
2. the result equals the same R ranks run in the one-process form on rank 0's GPU;
3. FusedOnPolicyRunner trains data-parallel, rank 0 writes a checkpoint, and every rank resumes from it.

    torchrun --nproc-per-node=2 tools/ppo_dp_check.py --out ok.txt      (rank 0 writes 'ok' to --out)
"""
import argparse
import os
import sys
import tempfile
from pathlib import Path

import torch
import torch.distributed as dist

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))


def main():
    ap = argparse.ArgumentParser(); ap.add_argument("--out", required=True); a = ap.parse_args()
    import test_ppo_dp_gpu as t
    import wheeledlab_b200 as wl
    from wheeledlab_b200.learner import FusedOnPolicyRunner, FusedPPO, PPOConfig, PPOExchange, update_local_ranks
    from wheeledlab_b200.runs import agent_cfg
    rank, local, world = int(os.environ["RANK"]), int(os.environ["LOCAL_RANK"]), int(os.environ["WORLD_SIZE"])
    torch.cuda.set_device(local); dev = f"cuda:{local}"
    dist.init_process_group("nccl", device_id=torch.device(dev))
    t.DEV = dev

    # 1-2: the update over peer memory, against the one-process form of the same ranks
    D, cfg = 14, PPOConfig(num_learning_epochs=2, num_mini_batches=4)
    blob, batches = t._synthetic(D, "elu", world, 4096, seed=11)      # every rank draws all R batches, keeps its own
    ppo = FusedPPO(blob.clone(), D, cfg, "elu", exchange=PPOExchange.symmetric(D, dev))
    ppo.update(*batches[rank])
    torch.cuda.synchronize()
    ppo.exchange.check()
    flat = torch.cat([ppo.blob, ppo.m, ppo.v, ppo.history.reshape(-1)])
    allp = [torch.empty_like(flat) for _ in range(world)]
    dist.all_gather(allp, flat)
    assert all(torch.equal(allp[0].view(torch.int32), q.view(torch.int32)) for q in allp), "replicas diverged"
    if rank == 0:
        ppos = [FusedPPO(blob.clone(), D, cfg, "elu", exchange=ex) for ex in PPOExchange.local(world, D, dev)]
        update_local_ranks(ppos, batches)
        assert torch.equal(ppos[0].blob.view(torch.int32), ppo.blob.view(torch.int32)), "multi-process != one-process form"
        assert torch.equal(ppos[0].v.view(torch.int32), ppo.v.view(torch.int32))

    # 3: the runner under torchrun, a checkpoint from rank 0, a resume on every rank
    log_dir = [tempfile.mkdtemp() if rank == 0 else None]
    dist.broadcast_object_list(log_dir, src=0)
    n = 512
    torch.manual_seed(0)
    env = wl.make("Isaac-MushrDriftRL-v0", device=dev, num_envs=n, seed=3, env_id_offset=rank * n)
    runner = FusedOnPolicyRunner(env, agent_cfg("elu", 16, 1), log_dir=log_dir[0], device=dev)
    runner.learn(2)
    allb = [torch.empty_like(runner.blob) for _ in range(world)]
    dist.all_gather(allb, runner.blob)
    assert all(torch.equal(allb[0].view(torch.int32), q.view(torch.int32)) for q in allb), "runner replicas diverged"
    dist.barrier()
    ckpt = Path(log_dir[0]) / "models" / "model_1.pt"
    assert ckpt.exists(), ckpt
    runner.load(str(ckpt))
    runner.learn(1)
    if rank == 0:
        Path(a.out).write_text("ok")
    dist.barrier(); dist.destroy_process_group()


if __name__ == "__main__":
    main()
