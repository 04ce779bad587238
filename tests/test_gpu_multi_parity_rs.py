"""ParityLocalCheckpointManager with parity_count = 2 on >= 3 GPUs (NCCL): saves over the fused P2P path and over NCCL with
stale bytes planted in the exchange buffer and the staging gaps, parity bytes against the host computation, m pack passes
and one combine launch per save, and two lost members rebuilt bit-exactly."""
import numpy as np
import pytest
import torch
import torch.distributed as dist

from _mp import run_ranks
from test_gpu_multi import bit_equal, flat_tensors, rank_state
from test_gpu_multi_parity import _image

pytestmark = [pytest.mark.gpu, pytest.mark.multigpu,
              pytest.mark.skipif(torch.cuda.device_count() < 3, reason="needs >= 3 CUDA devices")]


def _w_rs(rank, world, root, mode):
    import os
    import time

    os.environ["NVRX_B200_EXCHANGE"] = mode
    from nvidia_resiliency_ext.checkpointing.async_ckpt.core import AsyncCallsQueue
    from nvidia_resiliency_ext.checkpointing.b200 import erasure as E
    from nvidia_resiliency_ext.checkpointing.b200 import exchange as xch
    from nvidia_resiliency_ext.checkpointing.b200.engine import SnapshotEngine
    from nvidia_resiliency_ext.checkpointing.local.basic_state_dict import BasicTensorAwareStateDict
    from nvidia_resiliency_ext.checkpointing.local.ckpt_managers.parity_local_manager import ParityLocalCheckpointManager
    from nvidia_resiliency_ext.checkpointing.local.ckpt_managers.sharded_local_manager import shard_bytes_for

    m = 2
    mgr = ParityLocalCheckpointManager.from_replication_params(root, replication_jump=1, replication_factor=world, parity_count=m)
    code = mgr._code
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
        if it == 2:  # fused: m pack passes + one combine; NCCL: one pack + one combine
            assert engine.launches == launches0 + (1 if mode == "nccl" else m) + 1
        q.schedule_async_request(req)
        for t in live:
            t.zero_()
        assert q.maybe_finalize_async_calls(blocking=True, no_dist=False) == [it - 1]
    assert engine.last_exchange == ("nccl-alltoall-parity" if mode == "nccl" else "p2p-fused-parity")
    time.sleep(0.5)
    rs = f"iter_0000002_{rank}_local.rs{m}of{world}.pt"
    files = sorted(p.name for p in mgr.local_ckpt_dir.iterdir())
    assert files == sorted([f"iter_0000002_{rank}_local.pt", rs]), files

    states = {r: flat_tensors(rank_state(r + 20)) for r in range(world)}
    sb = shard_bytes_for(max(_image(states[r], 0)[1] for r in range(world)), code.k)
    want = []
    for p, s in enumerate(code.held_stripes(rank)):
        srcs = []
        for c in code.contributors(s):
            f = code.stripes_of(c).index(s)
            srcs.append(_image(states[c], code.k * sb)[0][f * sb : (f + 1) * sb])
        want.append(E.combine(code.G[p : p + 1], srcs)[0])
    spec = torch.load(mgr.local_ckpt_dir / rs, weights_only=False)
    assert spec["shard_bytes"] == sb and np.array_equal(spec["data"].numpy(), np.concatenate(want))
    dist.barrier()

    lost = [0, world - 1]
    if rank in lost:
        for p in mgr.local_ckpt_dir.iterdir():
            p.unlink()
    dist.barrier()
    mgr2 = ParityLocalCheckpointManager(root, clique=mgr.clique, parity_count=m)
    assert mgr2.find_latest() == 2
    loaded, cid = mgr2.load()
    got = list(loaded.tensors)
    assert cid == (2, rank, "") and len(got) == len(states[rank]) and all(a.is_cuda and bit_equal(a, b) for a, b in zip(got, states[rank]))
    q.close()


@pytest.mark.parametrize("mode", ["p2p", "nccl"])
def test_rs_manager_save_and_rebuild_two_lost(built_library, shm_dir, mode):
    run_ranks(_w_rs, min(torch.cuda.device_count(), 8), str(shm_dir / mode), mode, backend="nccl")
