"""ParityLocalCheckpointManager on >= 2 GPUs (NCCL): save over the fused P2P path and over NCCL, parity bytes against the
host computation with stale bytes planted in the exchange buffer and the staging gaps, one pack and one reduce launch per
save, one lost member rebuilt bit-exactly, and at F = 2 the parity equal to the striped fragment."""
import numpy as np
import pytest
import torch
import torch.distributed as dist

from _mp import run_ranks
from test_gpu_multi import bit_equal, flat_tensors, rank_state

pytestmark = [pytest.mark.gpu, pytest.mark.multigpu]


def _image(tensors, length):
    from nvidia_resiliency_ext.checkpointing.b200.engine import expected_layout

    nbytes = [t.numel() * t.element_size() for t in tensors]
    offs, _, total = expected_layout(nbytes, [False] * len(nbytes), 512)
    img = np.zeros(max(length, total), dtype=np.uint8)
    for t, off, nb in zip(tensors, offs, nbytes):
        if nb:
            img[off : off + nb] = t.detach().cpu().contiguous().view(-1).view(torch.uint8).numpy()
    return img, total


def _w_parity(rank, world, root, mode):
    import os
    import time

    os.environ["NVRX_B200_EXCHANGE"] = mode
    from nvidia_resiliency_ext.checkpointing.async_ckpt.core import AsyncCallsQueue
    from nvidia_resiliency_ext.checkpointing.b200 import exchange as xch
    from nvidia_resiliency_ext.checkpointing.b200.engine import SnapshotEngine
    from nvidia_resiliency_ext.checkpointing.local.basic_state_dict import BasicTensorAwareStateDict
    from nvidia_resiliency_ext.checkpointing.local.ckpt_managers.parity_local_manager import ParityLocalCheckpointManager
    from nvidia_resiliency_ext.checkpointing.local.ckpt_managers.sharded_local_manager import shard_bytes_for

    mgr = ParityLocalCheckpointManager.from_replication_params(root, replication_jump=1, replication_factor=world)
    n = world - 1
    q = AsyncCallsQueue(persistent=False)
    engine = SnapshotEngine.get()
    for it in (1, 2):
        if it == 2:  # stale bytes where no tensor is: the exchange buffer (as another exchange leaves it) and staging
            xch.as_uint8_tensor(engine._exchange_buf.ptr, engine._exchange_buf.nbytes, engine.device).fill_(0xAB)
            engine._exchange_dirty = True
            xch.as_uint8_tensor(engine._staging.ptr, engine._staging.nbytes, engine.device).fill_(0xCD)
            torch.cuda.synchronize()
            launches0 = engine.launches
        sd = BasicTensorAwareStateDict(rank_state(rank + 10 * it))
        live = list(sd.tensors)
        req = mgr.save(sd, it, is_async=True)
        if it == 2:
            assert engine.launches == launches0 + 2  # one pack, one reduce
        q.schedule_async_request(req)
        for t in live:
            t.zero_()
        assert q.maybe_finalize_async_calls(blocking=True, no_dist=False) == [it - 1]
    assert engine.last_exchange == ("nccl-alltoall-parity" if mode == "nccl" else "p2p-fused-parity")
    time.sleep(0.5)
    files = sorted(p.name for p in mgr.local_ckpt_dir.iterdir())
    assert files == sorted([f"iter_0000002_{rank}_local.pt", f"iter_0000002_{rank}_local.parity{n}.pt"]), files

    states = {m: flat_tensors(rank_state(m + 20)) for m in range(world)}
    sb = shard_bytes_for(max(_image(states[m], 0)[1] for m in range(world)), n)
    want = np.zeros(sb, dtype=np.uint8)
    for i in mgr._others(rank):
        k = mgr._others(i).index(rank)
        want ^= _image(states[i], n * sb)[0][k * sb : (k + 1) * sb]
    spec = torch.load(mgr.local_ckpt_dir / f"iter_0000002_{rank}_local.parity{n}.pt", weights_only=False)
    assert spec["shard_bytes"] == sb and np.array_equal(spec["data"].numpy(), want)
    dist.barrier()

    lost = world - 1
    if rank == lost:
        for p in mgr.local_ckpt_dir.iterdir():
            p.unlink()
    dist.barrier()
    mgr2 = ParityLocalCheckpointManager(root, clique=mgr.clique)
    assert mgr2.find_latest() == 2
    loaded, cid = mgr2.load()
    got = list(loaded.tensors)
    assert cid == (2, rank, "") and len(got) == len(states[rank]) and all(a.is_cuda and bit_equal(a, b) for a, b in zip(got, states[rank]))
    q.close()


@pytest.mark.parametrize("mode", ["p2p", "nccl"])
def test_parity_manager_save_and_rebuild(built_library, shm_dir, mode):
    run_ranks(_w_parity, min(torch.cuda.device_count(), 8), str(shm_dir / mode), mode, backend="nccl")


def _w_pair_equals_striped(rank, world, root):
    from nvidia_resiliency_ext.checkpointing.local.basic_state_dict import BasicTensorAwareStateDict
    from nvidia_resiliency_ext.checkpointing.local.ckpt_managers.parity_local_manager import ParityLocalCheckpointManager
    from nvidia_resiliency_ext.checkpointing.local.ckpt_managers.sharded_local_manager import ShardedLocalCheckpointManager

    par = ParityLocalCheckpointManager.from_replication_params(root + "/parity", replication_jump=1, replication_factor=2)
    par.save(BasicTensorAwareStateDict(rank_state(rank)), 1)
    striped = ShardedLocalCheckpointManager.from_replication_params(root + "/striped", replication_jump=1, replication_factor=2)
    striped.save(BasicTensorAwareStateDict(rank_state(rank)), 1)
    other = par._others(rank)[0]
    p = torch.load(par.local_ckpt_dir / f"iter_0000001_{rank}_local.parity1.pt", weights_only=False)["data"]
    f = torch.load(striped.local_ckpt_dir / f"iter_0000001_{other}_local.s0of1.pt", weights_only=False)["data"]
    assert torch.equal(p[: f.numel()], f) and int(p[f.numel():].count_nonzero()) == 0


def test_parity_pair_equals_striped_fragment(built_library, shm_dir):
    run_ranks(_w_pair_equals_striped, 2, str(shm_dir), backend="nccl")
