"""Replicated local checkpoints with the engine in the loop, on the CPU: real processes and real collectives (gloo), the
device replaced at the C-ABI boundary (tests/_fake_device.py).  Covers what tests/test_gpu_multi.py covers on GPUs -- save with
CliqueReplicationStrategy, lose a rank's files, find_latest, retrieve, restore -- for the default one-shot exchange and for the
modes written after the round's GPU budget was spent (streamed exchange, replicated zero-copy)."""
import os
import zipfile

import pytest
import torch

from _mp import run_ranks


def _rank_state(rank, wrap):
    g = torch.Generator().manual_seed(500 + rank)
    w = wrap if wrap is not None else (lambda t: t)
    return {
        "model": {"w": w(torch.randn(300 + 7 * rank, 129, generator=g)), "b": w(torch.randn(70_001 + rank, generator=g))},
        "opt": [{"m": w(torch.randn(4097, generator=g).to(torch.bfloat16)), "step": w(torch.tensor(float(rank)))}],
        "ids": w(torch.randint(0, 1 << 40, (1000 + rank,), generator=g)),
        "tag": f"rank{rank}",
    }


def _worker(rank, world, root, mode, zero_copy, kill):
    import torch.distributed as dist

    from _fake_device import FakeCudaTensor, fake_device, plain
    from oracle import snapshot_oracle as orc

    os.environ["NVRX_B200_EXCHANGE"] = mode
    os.environ["NVRX_B200_STREAM_CHUNK_MB"] = "0"  # 512-byte chunks: many ring turns
    if zero_copy:
        os.environ["NVRX_B200_ZERO_COPY"] = "1"
        os.environ["NVRX_B200_ZERO_COPY_REPLICAS"] = "1"
    mp = pytest.MonkeyPatch()
    try:
        with fake_device(mp) as (engine, lib):
            from nvidia_resiliency_ext.checkpointing.async_ckpt.core import AsyncCallsQueue
            from nvidia_resiliency_ext.checkpointing.b200 import exchange as xch
            from nvidia_resiliency_ext.checkpointing.local.basic_state_dict import BasicTensorAwareStateDict
            from nvidia_resiliency_ext.checkpointing.local.ckpt_managers.local_manager import LocalCheckpointManager
            from nvidia_resiliency_ext.checkpointing.local.replication.strategies import CliqueReplicationStrategy

            import ctypes as C

            def host_bytes(ptr, nbytes, device):
                return torch.frombuffer((C.c_uint8 * max(nbytes, 1)).from_address(ptr), dtype=torch.uint8)[:nbytes]

            class _S:
                cuda_stream = 0

                def synchronize(self):
                    pass

            mp.setattr(xch, "as_uint8_tensor", host_bytes)
            mp.setattr(torch.cuda, "current_stream", lambda *a, **k: _S())
            mp.setattr(torch.cuda, "ExternalStream", lambda *a, **k: None)
            mp.setattr(torch.cuda, "stream", lambda s: __import__("contextlib").nullcontext())
            mp.setattr(torch.cuda, "device_count", lambda: 1)

            strat = CliqueReplicationStrategy.from_replication_params(1, world)
            mgr = LocalCheckpointManager(root, repl_strategy=strat)
            q = AsyncCallsQueue(persistent=False)
            import time

            for it in (2, 3, 4, 5):  # steady state: later saves reuse geometry, views and (in zero-copy mode) freed slots
                time.sleep(0.4)  # let the background cleanup of the iteration before last finish (saves are minutes apart)
                dist.barrier()
                sd = BasicTensorAwareStateDict(_rank_state(rank + 10 * it, FakeCudaTensor.wrap))
                req = mgr.save(sd, it, is_async=True)
                assert sd.is_hollow
                q.schedule_async_request(req)
                assert q.maybe_finalize_async_calls(blocking=True, no_dist=False)
                assert engine.last_exchange == {"nccl": "nccl-allgather", "stream": "nccl-streamed"}[mode]
                # (the previous iteration's files are removed by a background thread: look at this iteration's only)
                files = sorted(p.name for p in mgr.local_ckpt_dir.iterdir() if p.name.startswith(f"iter_{it:07d}_"))
                assert files == sorted(f"iter_{it:07d}_{m}_local.pt" for m in range(world)), files
                for m in range(world):
                    path = mgr.local_ckpt_dir / f"iter_{it:07d}_{m}_local.pt"
                    tasd = torch.load(path, weights_only=False)
                    want = orc.flatten_tensors(_rank_state(m + 10 * it, None))
                    got = list(tasd.tensors)
                    assert len(got) == len(want)
                    for a, b in zip(got, want):
                        assert a.dtype == b.dtype and torch.equal(plain(a), b), (rank, m)
                    if zero_copy:
                        assert os.stat(path).st_nlink == 2, "replica file is expected to be a hard link to a slot"
                        with zipfile.ZipFile(path) as z:
                            assert z.testzip() is None, f"{path.name}: a record fails its CRC-32"
                assert len(engine._slots) <= engine.max_host_slots
            dist.barrier()
            if rank in kill:
                for p in mgr.local_ckpt_dir.iterdir():
                    p.unlink(missing_ok=True)  # the background cleanup of the previous iteration may get there first
            dist.barrier()
            mgr2 = LocalCheckpointManager(root, repl_strategy=strat)
            assert mgr2.find_latest() == 5
            loaded, cid = mgr2.load()
            assert cid == (5, rank, "")
            want = orc.flatten_tensors(_rank_state(rank + 50, None))
            got = list(loaded.tensors)
            assert len(got) == len(want) and all(a.is_cuda and torch.equal(plain(a), b) for a, b in zip(got, want))
            assert loaded.state_dict["tag"] == f"rank{rank + 50}"
            q.close()
    finally:
        mp.undo()


@pytest.mark.parametrize("mode,zero_copy", [("nccl", False), ("stream", False), ("nccl", True)])
def test_replicated_save_lose_a_rank_and_restore(shm_dir, built_library, mode, zero_copy):
    run_ranks(_worker, 2, str(shm_dir), mode, zero_copy, (1,), timeout=300)


def test_replicated_three_members_streamed(shm_dir, built_library):
    run_ranks(_worker, 3, str(shm_dir), "stream", False, (0, 2), timeout=300)


def _p2p_routing_worker(rank, world):
    """Rank 0 sends a state dict to rank 1 with isend_state_dict over gloo.  The packed exchange buffer looks like device
    memory here (as it is on a GPU): every tensor that reaches ``dist.send`` / ``dist.recv`` must be a host tensor, since
    gloo sends and receives host memory only."""
    import ctypes as C

    import torch.distributed as dist

    from _fake_device import FakeCudaTensor, fake_device, plain
    from oracle import snapshot_oracle as orc

    mp = pytest.MonkeyPatch()
    try:
        with fake_device(mp) as (engine, lib):
            from nvidia_resiliency_ext.checkpointing.b200 import exchange as xch
            from nvidia_resiliency_ext.checkpointing.local.basic_state_dict import BasicTensorAwareStateDict
            from nvidia_resiliency_ext.checkpointing.local.replication.group_utils import GroupWrapper

            def device_bytes(ptr, nbytes, device):
                return FakeCudaTensor.wrap(torch.frombuffer((C.c_uint8 * max(nbytes, 1)).from_address(ptr), dtype=torch.uint8)[:nbytes])

            def to(self, *args, **kwargs):
                dev = kwargs.get("device", args[0] if args else None)
                if isinstance(dev, (str, torch.device)) and torch.device(dev).type == "cpu":
                    return plain(self).clone()  # a device-to-host copy
                return FakeCudaTensor.wrap(torch.Tensor.to(plain(self), *args, **kwargs))

            class _S:
                cuda_stream = 0

                def synchronize(self):
                    pass

            seen = []

            def spy(real):
                def call(tensor, *args, **kwargs):
                    seen.append((real.__name__, tensor.is_cuda, tensor.numel()))
                    return real(plain(tensor), *args, **kwargs)

                return call

            mp.setattr(xch, "as_uint8_tensor", device_bytes)
            mp.setattr(FakeCudaTensor, "to", to, raising=False)
            mp.setattr(torch.cuda, "current_stream", lambda *a, **k: _S())
            mp.setattr(dist, "send", spy(dist.send))
            mp.setattr(dist, "recv", spy(dist.recv))

            gw = GroupWrapper()
            assert gw.backend == "gloo" and gw._payload_on_gpu()
            want = orc.flatten_tensors(_rank_state(0, None))
            if rank == 0:
                gw.isend_state_dict(BasicTensorAwareStateDict(_rank_state(0, FakeCudaTensor.wrap)), 1)
                assert lib.calls.count("pack") == 1
            else:
                got, log = gw.irecv_state_dict(0)
                tensors = list(got.tensors)
                assert lib.calls.count("scatter") == 1
                assert log["data_recv"] == sum(t.nbytes for t in want)
                assert len(tensors) == len(want)
                assert all(t.is_cuda and t.dtype == w.dtype and torch.equal(plain(t), w) for t, w in zip(tensors, want))
            payload = [s for s in seen if s[2] >= sum(t.nbytes for t in want)]
            assert [s[0] for s in payload] == ["send" if rank == 0 else "recv"], seen
            assert not any(is_cuda for _, is_cuda, _ in seen), f"a device tensor was handed to gloo: {seen}"
    finally:
        mp.undo()


def test_gloo_point_to_point_payload_goes_through_host_memory(built_library):
    """``send_packed`` / ``recv_packed`` on a gloo group (ranks sharing one GPU) copy the packed message through host memory."""
    run_ranks(_p2p_routing_worker, 2, timeout=300)


def _sharded_worker(rank, world, root, kill):
    import time

    import torch.distributed as dist

    from _fake_device import FakeCudaTensor, fake_device, plain
    from oracle import snapshot_oracle as orc

    os.environ["NVRX_B200_EXCHANGE"] = "nccl"
    mp = pytest.MonkeyPatch()
    try:
        with fake_device(mp) as (engine, lib):
            import ctypes as C

            from nvidia_resiliency_ext.checkpointing.async_ckpt.core import AsyncCallsQueue
            from nvidia_resiliency_ext.checkpointing.b200 import exchange as xch
            from nvidia_resiliency_ext.checkpointing.local.basic_state_dict import BasicTensorAwareStateDict
            from nvidia_resiliency_ext.checkpointing.local.ckpt_managers.sharded_local_manager import ShardedLocalCheckpointManager

            def host_bytes(ptr, nbytes, device):
                return torch.frombuffer((C.c_uint8 * max(nbytes, 1)).from_address(ptr), dtype=torch.uint8)[:nbytes]

            class _S:
                cuda_stream = 0

                def synchronize(self):
                    pass

            mp.setattr(xch, "as_uint8_tensor", host_bytes)
            mp.setattr(torch.cuda, "current_stream", lambda *a, **k: _S())
            mp.setattr(torch.cuda, "device_count", lambda: 1)
            mgr = ShardedLocalCheckpointManager.from_replication_params(root, replication_jump=1, replication_factor=world)
            q = AsyncCallsQueue(persistent=False)
            for it in (1, 2):
                req = mgr.save(BasicTensorAwareStateDict(_rank_state(rank + 10 * it, FakeCudaTensor.wrap)), it, is_async=True)
                q.schedule_async_request(req)
                q.maybe_finalize_async_calls(blocking=True, no_dist=False)
            time.sleep(0.5)
            n = world - 1
            files = sorted(p.name for p in mgr.local_ckpt_dir.iterdir())
            want = [f"iter_0000002_{rank}_local.pt"] + [f"iter_0000002_{m}_local.s{mgr._others(m).index(rank)}of{n}.pt" for m in range(world) if m != rank]
            assert files == sorted(want), (files, want)
            dist.barrier()
            if rank in kill:
                for p in mgr.local_ckpt_dir.iterdir():
                    p.unlink(missing_ok=True)  # the background cleanup of the previous iteration may get there first
            dist.barrier()
            mgr2 = ShardedLocalCheckpointManager(root, clique=mgr.clique)
            assert mgr2.find_latest() == 2
            loaded, cid = mgr2.load()
            want_t = orc.flatten_tensors(_rank_state(rank + 20, None))
            got = list(loaded.tensors)
            assert cid == (2, rank, "") and len(got) == len(want_t)
            assert all(a.is_cuda and a.dtype == b.dtype and torch.equal(plain(a), b) for a, b in zip(got, want_t))
            q.close()
    finally:
        mp.undo()


@pytest.mark.parametrize("world,kill", [(2, (1,)), (3, (0,))])
def test_striped_replicas_rebuild_a_lost_member(shm_dir, built_library, world, kill):
    """ShardedLocalCheckpointManager's device branch (pack + all_to_all of fragments, rebuild by all-gathering them back)."""
    run_ranks(_sharded_worker, world, str(shm_dir), kill, timeout=300)
