"""Caller-side demo (what reference examples/checkpointing/local_ckpt.py and async_ckpt.py do): the user code imports
``nvidia_resiliency_ext.checkpointing...`` exactly as with the reference; only ``sys.path`` decides which package runs.

    torchrun --standalone --local-addr 127.0.0.1 --nproc-per-node 2 examples/local_ckpt_demo.py --replication [--sharded]
"""
import argparse
import os
import shutil
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent.parent / "nvidia-resiliency-ext_b200"))

import torch
import torch.distributed as dist
import torch.nn as nn

from nvidia_resiliency_ext.checkpointing.async_ckpt.core import AsyncCallsQueue
from nvidia_resiliency_ext.checkpointing.async_ckpt.torch_ckpt import TorchAsyncCheckpoint
from nvidia_resiliency_ext.checkpointing.local.basic_state_dict import BasicTensorAwareStateDict
from nvidia_resiliency_ext.checkpointing.local.ckpt_managers.local_manager import LocalCheckpointManager
from nvidia_resiliency_ext.checkpointing.local.replication.strategies import CliqueReplicationStrategy


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ckpt_dir", default="/dev/shm/nvrx_b200_demo")
    ap.add_argument("--replication", action="store_true")
    ap.add_argument("--sharded", action="store_true", help="striped fragments instead of full replicas (extension of this package)")
    args = ap.parse_args()
    rank, world, local = (int(os.environ.get(k, d)) for k, d in (("RANK", "0"), ("WORLD_SIZE", "1"), ("LOCAL_RANK", "0")))
    torch.cuda.set_device(local)
    dist.init_process_group("nccl")
    model = nn.Sequential(nn.Linear(1024, 4096), nn.ReLU(), nn.Linear(4096, 1024)).cuda()
    opt = torch.optim.Adam(model.parameters())
    model(torch.randn(8, 1024, device="cuda")).sum().backward()
    opt.step()

    # 1. async torch.save of a plain state dict
    ckpt = TorchAsyncCheckpoint()
    path = Path(args.ckpt_dir) / f"global_{rank}.pt"
    path.parent.mkdir(parents=True, exist_ok=True)
    ckpt.async_save(model.state_dict(), path)          # returns after enqueueing pack + drain
    ckpt.finalize_async_save(blocking=True)
    assert all(torch.equal(v.cpu(), model.state_dict()[k].cpu()) for k, v in torch.load(path).items())
    ckpt.close()

    # 2. local checkpoint manager (+ replication)
    if args.sharded:
        from nvidia_resiliency_ext.checkpointing.local.ckpt_managers.sharded_local_manager import ShardedLocalCheckpointManager

        mgr = ShardedLocalCheckpointManager.from_replication_params(args.ckpt_dir, replication_jump=1, replication_factor=world)
    else:
        strat = CliqueReplicationStrategy.from_replication_params(1, world) if args.replication and world > 1 else None
        mgr = LocalCheckpointManager(args.ckpt_dir, repl_strategy=strat)
    queue = AsyncCallsQueue(persistent=False)
    for iteration in (10, 20):
        sd = {"model": model.state_dict(), "optimizer": opt.state_dict()["state"], "iteration": iteration}
        queue.schedule_async_request(mgr.save(BasicTensorAwareStateDict(sd), iteration, is_async=True))
        model(torch.randn(8, 1024, device="cuda")).sum().backward()   # training continues while the snapshot drains
        opt.step()
        queue.maybe_finalize_async_calls(blocking=True, no_dist=False)
    assert mgr.find_latest() == 20
    loaded, ckpt_id = mgr.load()
    print(f"rank {rank}: restored {ckpt_id} with {len(list(loaded.tensors))} tensors on {next(iter(loaded.tensors)).device}")
    queue.close()
    dist.barrier()
    if rank == 0:
        shutil.rmtree(args.ckpt_dir, ignore_errors=True)
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
