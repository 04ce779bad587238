"""Multi-GPU rows of the hot path (NCCL over NVLink): packed replica exchange, replicated save, retrieval of a lost
shard + scatter restore.  Needs >= 2 GPUs (``gpurun --gpus 2``); world sizes follow the GPUs present (max 8)."""
import hashlib

import numpy as np
import pytest
import torch
import torch.distributed as dist

from _mp import run_ranks

pytestmark = [pytest.mark.gpu, pytest.mark.multigpu]


def bit_equal(a, b):
    a, b = a.detach().cpu(), b.detach().cpu()
    return a.dtype == b.dtype and a.shape == b.shape and (a.numel() == 0 or torch.equal(a.contiguous().view(-1).view(torch.uint8), b.contiguous().view(-1).view(torch.uint8)))


def rank_state(rank, device="cuda"):
    g = torch.Generator(device=device).manual_seed(500 + rank)
    flat = torch.randn(200_003, device=device, generator=g)
    return {
        "model": {"w": torch.randn(300 + 7 * rank, 129, device=device, generator=g), "view": flat[1 : 1 + 70_001 + rank]},
        "opt": [{"m": torch.randn(4097, device=device, generator=g).to(torch.bfloat16), "step": torch.tensor(float(rank), device=device)}],
        "ids": torch.randint(0, 1 << 40, (1000 + rank,), device=device, generator=g),
        "tag": f"rank{rank}",
    }


def flat_tensors(sd):
    out = []

    def walk(x):
        for v in (x.values() if isinstance(x, dict) else x):
            if isinstance(v, (dict, list)):
                walk(v)
            elif isinstance(v, torch.Tensor):
                out.append(v)

    walk(sd)
    return out


def edge_state(seed, shrink=False, device="cuda"):
    """``rank_state`` plus a short odd-length bf16 vector and an empty tensor; ``shrink``: a smaller image than the same
    seed's full state (one tensor gone, another shorter), so that bytes of a larger earlier save lie past its end."""
    sd = rank_state(seed, device)
    g = torch.Generator(device=device).manual_seed(900 + seed)
    sd["edge"] = {"odd": torch.randn(7 + 2 * (seed % 5), device=device, generator=g).to(torch.bfloat16),
                  "empty": torch.empty(0, 3, device=device)}
    if shrink:
        del sd["ids"]
        sd["model"]["w"] = sd["model"]["w"][: 40 + seed % 13].clone()
    return sd


def _image(tensors, length):
    from nvidia_resiliency_ext.checkpointing.b200.engine import expected_layout

    nbytes = [t.numel() * t.element_size() for t in tensors]
    offs, _, total = expected_layout(nbytes, [False] * len(nbytes), 512)
    img = np.zeros(max(length, total), dtype=np.uint8)
    for t, off, nb in zip(tensors, offs, nbytes):
        if nb:
            img[off : off + nb] = t.detach().cpu().contiguous().view(-1).view(torch.uint8).numpy()
    return img, total


def _covered(tensors):
    """Which bytes of the packed image of ``tensors`` belong to a tensor (not to a gap or the padding)."""
    from nvidia_resiliency_ext.checkpointing.b200.engine import expected_layout

    nbytes = [t.numel() * t.element_size() for t in tensors]
    offs, _, total = expected_layout(nbytes, [False] * len(nbytes), 512)
    mask = np.zeros(total, dtype=bool)
    for off, nb in zip(offs, nbytes):
        mask[off : off + nb] = True
    return mask


def fill_staging(engine, value):
    """Stale bytes all over the engine's staging (grown first, so that a later save or rebuild does not get a fresh one)."""
    from nvidia_resiliency_ext.checkpointing.b200 import exchange as xch

    st = engine._ensure_staging(16 << 20)
    xch.as_uint8_tensor(st.ptr, st.nbytes, engine.device).fill_(value)
    torch.cuda.synchronize()


def _w_allgather_batch(rank, world, mode):
    import os

    os.environ["NVRX_B200_EXCHANGE"] = mode
    from nvidia_resiliency_ext.checkpointing.b200.engine import SnapshotEngine
    from nvidia_resiliency_ext.checkpointing.local.replication.group_utils import GroupWrapper

    gw = GroupWrapper()
    mine = flat_tensors(rank_state(rank))
    launches0 = SnapshotEngine.get().launches
    got = gw.all_gather_batch(mine, target_device="cpu")
    assert SnapshotEngine.get().launches == launches0 + 1  # ONE pack kernel; the reference does world*N broadcasts
    assert SnapshotEngine.get().last_exchange == {"nccl": "nccl-allgather", "p2p": "p2p-fused", "stream": "nccl-streamed"}[mode]
    for s in gw.last_snapshots:
        s.wait()
    assert len(got) == world
    for r in range(world):
        want = flat_tensors(rank_state(r))
        assert len(got[r]) == len(want)
        for a, b in zip(got[r], want):
            assert not a.is_cuda and bit_equal(a, b), (rank, r)
    for s in gw.last_snapshots:
        s.release()
    # device-resident variant
    got = gw.all_gather_batch(mine, target_device=None)
    for r in range(world):
        for a, b in zip(got[r], flat_tensors(rank_state(r))):
            assert a.is_cuda and bit_equal(a, b)




def _w_allgather_streamed_small_chunks(rank, world):
    import os

    os.environ["NVRX_B200_STREAM_CHUNK_MB"] = "0"  # -> 512-byte chunks: many ring turns even for the small test state
    _w_allgather_batch(rank, world, "stream")


def test_all_gather_batch_streamed_exchange(built_library):
    """NVRX_B200_EXCHANGE=stream: pack on the training stream, chunked all-gather + drain in the background."""
    world = min(torch.cuda.device_count(), 8)
    run_ranks(_w_allgather_batch, world, "stream", backend="nccl")
    run_ranks(_w_allgather_streamed_small_chunks, world, backend="nccl", timeout=600)


@pytest.mark.parametrize("mode", ["p2p", "nccl"])
def test_all_gather_batch_packed_exchange(built_library, mode):
    """p2p: pack fused with the all-gather (NVLink peer stores from the pack kernel); nccl: pack + one NCCL all-gather."""
    run_ranks(_w_allgather_batch, min(torch.cuda.device_count(), 8), mode, backend="nccl")


def _w_replicated_save_and_restore(rank, world, root, jump, factor, kill):
    from nvidia_resiliency_ext.checkpointing.async_ckpt.core import AsyncCallsQueue
    from nvidia_resiliency_ext.checkpointing.local.basic_state_dict import BasicTensorAwareStateDict
    from nvidia_resiliency_ext.checkpointing.local.ckpt_managers.local_manager import LocalCheckpointManager
    from nvidia_resiliency_ext.checkpointing.local.replication.strategies import CliqueReplicationStrategy

    strat = CliqueReplicationStrategy.from_replication_params(jump, factor)
    mgr = LocalCheckpointManager(root, repl_strategy=strat)
    q = AsyncCallsQueue(persistent=False)
    sd = BasicTensorAwareStateDict(rank_state(rank))
    live = list(sd.tensors)
    req = mgr.save(sd, 4, is_async=True)
    assert sd.is_hollow  # reference contract: replicate() leaves the input hollow (strategies.py:139)
    q.schedule_async_request(req)
    for t in live:
        t.zero_()  # training goes on
    assert q.maybe_finalize_async_calls(blocking=True, no_dist=False) == [0]
    members = strat.local_group.ranks
    files = sorted(p.name for p in mgr.local_ckpt_dir.iterdir())
    assert files == sorted(f"iter_0000004_{m}_local.pt" for m in members), files
    # every replica file holds the owner's bits
    for m in members:
        tasd = torch.load(mgr.local_ckpt_dir / f"iter_0000004_{m}_local.pt", weights_only=False)
        assert all(bit_equal(a, b) for a, b in zip(tasd.tensors, flat_tensors(rank_state(m))))
    dist.barrier()
    if rank in kill:
        for p in mgr.local_ckpt_dir.iterdir():
            p.unlink()
    dist.barrier()
    mgr2 = LocalCheckpointManager(root, repl_strategy=strat)
    assert mgr2.find_latest() == 4
    loaded, cid = mgr2.load()
    assert cid == (4, rank, "")
    want = flat_tensors(rank_state(rank))
    got = list(loaded.tensors)
    assert len(got) == len(want) and all(a.is_cuda and bit_equal(a, b) for a, b in zip(got, want))
    assert loaded.state_dict["tag"] == f"rank{rank}"
    q.close()


def test_replicated_save_retrieve_restore_pairs(built_library, shm_dir):
    world = 2
    run_ranks(_w_replicated_save_and_restore, world, str(shm_dir), 1, 2, (1,), backend="nccl")


def _w_replicated_zero_copy(rank, world, root, jump, factor, kill):
    import os

    os.environ["NVRX_B200_ZERO_COPY_REPLICAS"] = "1"
    os.environ["NVRX_B200_ZERO_COPY"] = "1"  # on every member: the container geometry of a slice is computed by all of them
    _w_replicated_save_and_restore(rank, world, root, jump, factor, kill)
    # every surviving file on this rank is a hard link to one of its pinned slots, not a copy
    from pathlib import Path

    files = [p for p in Path(root).rglob("iter_*_local.pt")]
    mine = [p for p in files if f"/{rank}/" in str(p)]
    assert rank in kill or (mine and all(os.stat(p).st_nlink == 2 for p in mine)), [(str(p), os.stat(p).st_nlink) for p in mine]


def test_replicated_save_zero_copy_pairs(built_library, shm_dir):
    """Replicated zero-copy (written after round 1's GPU budget was spent): each member's slice of the exchange buffer is
    drained into a slot of its own in container geometry and published as that member's file."""
    run_ranks(_w_replicated_zero_copy, 2, str(shm_dir), 1, 2, (1,), backend="nccl")


def test_replicated_save_retrieve_restore_full_clique(built_library, shm_dir):
    world = min(torch.cuda.device_count(), 8)
    if world < 4:
        pytest.skip("needs >= 4 GPUs")
    run_ranks(_w_replicated_save_and_restore, world, str(shm_dir), 1, world, tuple(range(1, world)), backend="nccl", timeout=600)


def _w_sharded(rank, world, root, mode, jump, factor, positions):
    """Saves of ShardedLocalCheckpointManager on the device path, own file and every held fragment checked byte for byte,
    then each lost set in ``positions`` (indices into the clique, the same in every clique) rebuilt from the fragments,
    with a new save between them."""
    import os
    import time

    os.environ["NVRX_B200_EXCHANGE"] = mode
    from nvidia_resiliency_ext.checkpointing.async_ckpt.core import AsyncCallsQueue
    from nvidia_resiliency_ext.checkpointing.b200.engine import SnapshotEngine
    from nvidia_resiliency_ext.checkpointing.local.basic_state_dict import BasicTensorAwareStateDict
    from nvidia_resiliency_ext.checkpointing.local.ckpt_managers.sharded_local_manager import ShardedLocalCheckpointManager, fragment_range

    mgr = ShardedLocalCheckpointManager.from_replication_params(root, replication_jump=jump, replication_factor=factor)
    members = mgr._members
    n = len(members) - 1
    branch = "nccl-alltoall" if mode == "nccl" else "p2p-fused-sharded"
    q = AsyncCallsQueue(persistent=False)
    engine = SnapshotEngine.get()

    def save(man, it):
        sd = BasicTensorAwareStateDict(edge_state(10 * it + rank))
        live = list(sd.tensors)
        launches0 = engine.launches
        req = man.save(sd, it, is_async=True)
        assert engine.last_exchange == branch and engine.launches == launches0 + 1, (engine.last_exchange, engine.launches - launches0)
        q.schedule_async_request(req)
        for t in live:
            t.zero_()  # training goes on: the files must hold the state from before
        assert len(q.maybe_finalize_async_calls(blocking=True, no_dist=False)) == 1

    def want(r, it):
        return flat_tensors(edge_state(10 * it + r))

    for it in (1, 2):
        save(mgr, it)
    time.sleep(0.5)
    files = sorted(p.name for p in mgr.local_ckpt_dir.iterdir())
    expect = [f"iter_0000002_{rank}_local.pt"] + [f"iter_0000002_{m}_local.s{mgr._others(m).index(rank)}of{n}.pt" for m in members if m != rank]
    assert files == sorted(expect), (files, expect)
    own = list(torch.load(mgr.local_ckpt_dir / f"iter_0000002_{rank}_local.pt", weights_only=False).tensors)
    assert len(own) == len(want(rank, 2)) and all(bit_equal(a, b) for a, b in zip(own, want(rank, 2))), "own file"
    for m in members:
        if m == rank:
            continue
        k = mgr._others(m).index(rank)
        img, total = _image(want(m, 2), 0)
        spec = torch.load(mgr.local_ckpt_dir / f"iter_0000002_{m}_local.s{k}of{n}.pt", weights_only=False)
        lo, hi = fragment_range(total, spec["shard_bytes"], k)
        tensor_bytes = _covered(want(m, 2))[lo:hi]  # striped fragments need not clear the gaps: only tensor bytes count
        assert spec["total_bytes"] == total and spec["data"].numel() == hi - lo, ("fragment size", m, k)
        assert np.array_equal(spec["data"].numpy()[tensor_bytes], img[lo:hi][tensor_bytes]), ("fragment bytes", m, k)
    dist.barrier()

    it = 2
    for pos in positions:
        lost = [members[i] for i in pos]
        if rank in lost:
            for p in mgr.local_ckpt_dir.glob(f"iter_{it:07d}_*"):
                p.unlink()
        dist.barrier()
        fill_staging(engine, 0xCD)  # the rebuilt image must not keep staging's bytes
        probe = ShardedLocalCheckpointManager(root, clique=mgr.clique)
        assert probe.find_latest() == it
        loaded, cid = probe.load()
        got = list(loaded.tensors)
        ref = want(rank, it)
        assert cid == (it, rank, "") and len(got) == len(ref), (lost, rank)
        assert all(a.is_cuda and bit_equal(a, b) for a, b in zip(got, ref)), ("rebuild", lost, rank)
        dist.barrier()
        it += 1
        save(probe, it)
        mgr = probe
    q.close()


@pytest.mark.parametrize("mode", ["p2p", "nccl"])
def test_sharded_manager_all_to_all_and_rebuild(built_library, shm_dir, mode):
    """North-star layout: 1/(F-1) fragments exchanged with one all-to-all (fused into the pack kernel over NVLink P2P, or
    NCCL), a member that lost its storage is rebuilt from the fragments with the scatter kernel, bit-exact."""
    world = min(torch.cuda.device_count(), 8)
    run_ranks(_w_sharded, world, str(shm_dir / mode), mode, 1, world, [(world - 1,)], backend="nccl")
