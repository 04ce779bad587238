"""Multi-GPU rows of the hot path (NCCL over NVLink): packed replica exchange, replicated save, retrieval of a lost
shard + scatter restore.  Needs >= 2 GPUs; world sizes follow the GPUs present (max 8).  The workers
are shared with ``test_gpu_one_device_cliques`` and ``test_gpu_one_device_replication``, which run them on one GPU."""
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


def wipe(t):
    """Zero every byte of ``t``'s storage (a view's base included)."""
    torch.empty(0, dtype=torch.uint8, device=t.device).set_(t.untyped_storage()).zero_()


def host_copy(sd):
    """The tensors of ``sd`` as host tensors: the plain reference a save is compared with.  The device copies are wiped
    before they are freed, so that a later allocation (a receive buffer, say) cannot find the expected bytes left behind in
    the caching allocator and pass without being written."""
    out = []
    for t in flat_tensors(sd):
        out.append(t.cpu())
        wipe(t)
    return out


def host_state(seed, shrink=False):
    return host_copy(edge_state(seed, shrink))


def _w_allgather_batch(rank, world, mode, small_chunks=False):
    """``GroupWrapper.all_gather_batch`` of ``edge_state`` in exchange ``mode`` (``NVRX_B200_EXCHANGE``), to a CPU target and
    to the device: one pack launch each, the branch that ran, and every member's tensors bit for bit on every rank.  The
    live tensors are zeroed on the training stream right after the call.  ``small_chunks``: 512-byte chunks for the
    streamed exchange, many turns of its ring."""
    import os

    os.environ["NVRX_B200_EXCHANGE"] = mode
    if small_chunks:
        os.environ["NVRX_B200_STREAM_CHUNK_MB"] = "0"
    from nvidia_resiliency_ext.checkpointing.b200 import exchange as xch
    from nvidia_resiliency_ext.checkpointing.b200.engine import SnapshotEngine
    from nvidia_resiliency_ext.checkpointing.local.replication.group_utils import GroupWrapper

    if small_chunks:
        assert xch.stream_schedule(1 << 20, xch.STREAM_CHUNK)[0] == 512
    engine = SnapshotEngine.get()
    gw = GroupWrapper()
    want = [host_state(r) for r in range(world)]
    for target, branch in (("cpu", {"nccl": "nccl-allgather", "p2p": "p2p-fused", "stream": "nccl-streamed"}[mode]),
                           (None, "nccl-allgather" if mode == "nccl" else "p2p-fused")):
        mine = flat_tensors(edge_state(rank))
        launches0 = engine.launches
        got = gw.all_gather_batch(mine, target_device=target)
        assert engine.launches == launches0 + 1, ("launches", target, engine.launches - launches0)  # ONE pack kernel; the reference does world*N broadcasts
        assert engine.last_exchange == branch, (target, engine.last_exchange)
        for t in mine:
            t.zero_()  # training goes on
        for s in gw.last_snapshots:
            s.wait()
        assert len(got) == world
        for r in range(world):
            assert len(got[r]) == len(want[r]), (target, rank, r)
            for i, (a, b) in enumerate(zip(got[r], want[r])):
                assert a.is_cuda == (target is None) and bit_equal(a, b), ("all_gather_batch", target, rank, r, i)
        for s in gw.last_snapshots:
            s.release()


def count_launches(engine):
    """Wrap ``send_packed`` / ``recv_packed``: every call appends the kernels it launched to ``calls["send" / "recv"]``."""
    from nvidia_resiliency_ext.checkpointing.b200 import exchange as xch

    calls = {"send": [], "recv": []}
    for kind, log in calls.items():
        def wrapped(*args, _real=getattr(xch, f"{kind}_packed"), _log=log, **kwargs):
            before = engine.launches
            _real(*args, **kwargs)
            _log.append(engine.launches - before)

        setattr(xch, f"{kind}_packed", wrapped)
    return calls


def check_replicas(mgr, it, states, zero_copy=False, lost=()):
    """Every ``iter_<it>_<m>_local.pt`` in this rank's directory holds member m's state bit for bit (none where this rank
    lost its files); with zero-copy replicas each is also a hard link to a slot and passes zipfile's CRC check."""
    import os
    import zipfile

    files = sorted(p.name for p in mgr.local_ckpt_dir.iterdir() if p.name.startswith(f"iter_{it:07d}_"))
    want = [] if mgr.rank in lost else sorted(f"iter_{it:07d}_{m}_local.pt" for m in states)
    assert files == want, (it, files)
    for name in files:
        m = int(name.split("_")[2])
        path = mgr.local_ckpt_dir / name
        got = list(torch.load(path, weights_only=False).tensors)
        assert len(got) == len(states[m]) and all(bit_equal(a, b) for a, b in zip(got, states[m])), ("replica file", it, m)
        if zero_copy:
            assert os.stat(path).st_nlink == 2, ("not a hard link to a slot", name, os.stat(path).st_nlink)
            with zipfile.ZipFile(path) as zf:
                assert zf.testzip() is None, f"{name}: a record fails its CRC-32"


def _w_replicated(rank, world, root, mode, jump, factor, kills, restructure=False, zero_copy=False):
    """LocalCheckpointManager with CliqueReplicationStrategy(jump, factor) in exchange ``mode``: saves of ``edge_state``
    (``restructure``: a full state, a smaller one, then a larger one, so that the exchange buffer and the peer maps are
    regenerated), every replica file on every member checked against the owner's state after each save, then for each
    position tuple in ``kills`` (indices into the clique, the same in every clique) those members lose their files and a
    fresh manager retrieves every rank's shard bit for bit onto the device, with a new save between the kill sets."""
    import os

    os.environ["NVRX_B200_EXCHANGE"] = mode
    if zero_copy:
        os.environ["NVRX_B200_ZERO_COPY_REPLICAS"] = "1"
        os.environ["NVRX_B200_ZERO_COPY"] = "1"  # on every member: the container geometry of a slice is computed by all of them
        os.environ["NVRX_B200_ZIP_CRC"] = "1"
    from nvidia_resiliency_ext.checkpointing.async_ckpt.core import AsyncCallsQueue
    from nvidia_resiliency_ext.checkpointing.b200.engine import SnapshotEngine
    from nvidia_resiliency_ext.checkpointing.local.basic_state_dict import BasicTensorAwareStateDict
    from nvidia_resiliency_ext.checkpointing.local.ckpt_managers.local_manager import LocalCheckpointManager
    from nvidia_resiliency_ext.checkpointing.local.replication.strategies import CliqueReplicationStrategy

    strat = CliqueReplicationStrategy.from_replication_params(jump, factor)
    members = list(strat.local_group.ranks)
    branch = {"nccl": "nccl-allgather", "p2p": "p2p-fused"}.get(mode)
    engine = SnapshotEngine.get()
    q = AsyncCallsQueue(persistent=False)
    states = {}

    def save(man, it, shrink=False):
        states[it] = {m: host_state(10 * it + m, shrink) for m in members}
        sd = BasicTensorAwareStateDict(edge_state(10 * it + rank, shrink))
        live = list(sd.tensors)
        launches0 = engine.launches
        req = man.save(sd, it, is_async=True)
        assert sd.is_hollow  # reference contract: replicate() leaves the input hollow (strategies.py:139)
        assert engine.launches == launches0 + 1, ("launches", it, engine.launches - launches0)  # one pack for the clique
        assert branch is None or engine.last_exchange == branch, engine.last_exchange
        idx = q.schedule_async_request(req)
        for t in live:
            t.zero_()  # training goes on: the files must hold the state from before
        assert q.maybe_finalize_async_calls(blocking=True, no_dist=False) == [idx]
        check_replicas(man, it, states[it], zero_copy)

    mgr = LocalCheckpointManager(root, repl_strategy=strat)
    it = 1
    save(mgr, it)
    if restructure:
        it += 1
        save(mgr, it, shrink=True)
        before = engine._exchange_buf.nbytes
        it += 1
        save(mgr, it)  # larger than the first save: every member regenerates its buffer and re-imports the peers'
        assert engine._exchange_buf.nbytes > before, (before, engine._exchange_buf.nbytes)

    calls = count_launches(engine)
    for n, pos in enumerate(kills):
        lost = [members[i] for i in pos]
        dist.barrier()
        if rank in lost:
            for p in mgr.local_ckpt_dir.glob(f"iter_{it:07d}_*"):
                p.unlink()
        dist.barrier()
        fill_staging(engine, 0xCD)  # the restored tensors must not keep staging's bytes
        calls["send"].clear()
        calls["recv"].clear()
        probe = LocalCheckpointManager(root, repl_strategy=strat)
        assert probe.find_latest() == it
        loaded, cid = probe.load()
        assert cid == (it, rank, "")
        got = list(loaded.tensors)
        want = states[it][rank]
        assert len(got) == len(want) and all(a.is_cuda and bit_equal(a, b) for a, b in zip(got, want)), ("retrieve", lost, rank)
        assert loaded.state_dict["tag"] == f"rank{10 * it + rank}"
        # one pack per message sent, one scatter per message received; a lost member receives its shard once
        assert calls["recv"] == ([1] if rank in lost else []), ("receives", lost, calls["recv"])
        assert all(n_launch == 1 for n_launch in calls["send"]), ("sends", calls["send"])
        assert sum(len(c) for c in strat.local_group.all_gather_object(calls["send"])) == len(lost)
        check_replicas(mgr, it, states[it], zero_copy, lost)
        dist.barrier()
        if n + 1 < len(kills):
            it += 1
            save(probe, it)
        mgr = probe
    q.close()


def _w_replicated_held(rank, world, root, mode, cycles_per_ms):
    """Back-to-back replicated saves with save N's drain held open by a sleep kernel at the head of ``_side`` on every
    rank.  ``p2p``: save N+1 is issued while save N's drain is still queued, and its pack must wait for that drain before
    it stores into the exchange buffers (``_exchange_free``).  ``stream`` (512-byte chunks): the ring turns back to a half
    while the drains out of it are held, and each all-gather into that half must wait for them (``half_free``); gloo's
    host-blocking all-gather makes save N itself wait there, so the window is asserted at that all-gather.  Both files
    must hold their own states."""
    import os

    os.environ["NVRX_B200_EXCHANGE"] = mode
    os.environ["NVRX_B200_STREAM_CHUNK_MB"] = "0"
    from nvidia_resiliency_ext.checkpointing.async_ckpt.core import AsyncCallsQueue
    from nvidia_resiliency_ext.checkpointing.b200.engine import SnapshotEngine
    from nvidia_resiliency_ext.checkpointing.local.basic_state_dict import BasicTensorAwareStateDict
    from nvidia_resiliency_ext.checkpointing.local.ckpt_managers.local_manager import LocalCheckpointManager
    from nvidia_resiliency_ext.checkpointing.local.replication.strategies import CliqueReplicationStrategy
    from test_gpu_handoffs import assert_open, hold, queued_after

    strat = CliqueReplicationStrategy.from_replication_params(1, world)
    members = list(strat.local_group.ranks)
    engine = SnapshotEngine.get()
    q = AsyncCallsQueue(persistent=False)
    mgr = LocalCheckpointManager(root, repl_strategy=strat)
    mgr._cleanup = lambda iteration: None  # keep save N's files after save N+1 is finalized: both are checked

    def state(it, r):
        """Member r's state of save ``it``: one structure for every save (plans, buffers and slots are reused inside the
        window), other bytes."""
        sd = edge_state(r)
        for t in flat_tensors(sd):
            t.add_(it)
        return sd

    def issue(it):
        sd = BasicTensorAwareStateDict(state(it, rank))
        live = list(sd.tensors)
        req = mgr.save(sd, it, is_async=True)
        for t in live:
            t.zero_()
        return req

    def finish(reqs):
        idx = [q.schedule_async_request(r) for r in reqs]
        assert q.maybe_finalize_async_calls(blocking=True, no_dist=False) == idx

    # the references first: computed inside the window they would take part of it
    states = {it: {m: host_copy(state(it, m)) for m in members} for it in (1, 2, 3, 4)}
    # warm-up outside any hold: the sleep and exchange kernels loaded, two host slots created and pinned, the ring built
    hold(engine._side.handle, cycles_per_ms, 1)
    finish([issue(1), issue(2)])
    for it in (1, 2):
        check_replicas(mgr, it, states[it])
    ring_gathers, real_gather = [], dist.all_gather_into_tensor

    def gather(out, *args, **kwargs):
        if out.is_cuda:  # the ring's all-gathers (all_gather_int runs on the CPU over gloo)
            ring_gathers.append(mark.query())
        return real_gather(out, *args, **kwargs)

    hold(engine._side.handle, cycles_per_ms)
    mark = queued_after(engine._side.handle)
    dist.all_gather_into_tensor = gather
    try:
        first = issue(3)
    finally:
        dist.all_gather_into_tensor = real_gather
    if mode == "stream":
        assert engine.last_exchange == "nccl-streamed"
        # chunk 2 is the first all-gather into ring half 0 again: it was issued while chunk 0's drain was still held
        assert len(ring_gathers) > 2 and ring_gathers[2] is False, ("the window was closed", ring_gathers[:4])
    else:
        assert engine.last_exchange == "p2p-fused"
        assert_open(mark)
    second = issue(4)
    finish([first, second])
    for it in (3, 4):
        check_replicas(mgr, it, states[it])
    q.close()


def test_all_gather_batch_streamed_exchange(built_library):
    """NVRX_B200_EXCHANGE=stream: pack on the training stream, chunked all-gather + drain in the background."""
    world = min(torch.cuda.device_count(), 8)
    run_ranks(_w_allgather_batch, world, "stream", backend="nccl")
    run_ranks(_w_allgather_batch, world, "stream", True, backend="nccl", timeout=600)


@pytest.mark.parametrize("mode", ["p2p", "nccl"])
def test_all_gather_batch_packed_exchange(built_library, mode):
    """p2p: pack fused with the all-gather (NVLink peer stores from the pack kernel); nccl: pack + one NCCL all-gather."""
    run_ranks(_w_allgather_batch, min(torch.cuda.device_count(), 8), mode, backend="nccl")


def test_replicated_save_retrieve_restore_pairs(built_library, shm_dir):
    run_ranks(_w_replicated, 2, str(shm_dir), "auto", 1, 2, [(1,)], backend="nccl")


def test_replicated_save_zero_copy_pairs(built_library, shm_dir):
    """Replicated zero-copy: each member's slice of the exchange buffer is drained into a slot of its own in container
    geometry and published as that member's file."""
    run_ranks(_w_replicated, 2, str(shm_dir), "auto", 1, 2, [(1,)], False, True, backend="nccl")


def test_replicated_save_retrieve_restore_full_clique(built_library, shm_dir):
    world = min(torch.cuda.device_count(), 8)
    if world < 4:
        pytest.skip("needs >= 4 GPUs")
    run_ranks(_w_replicated, world, str(shm_dir), "auto", 1, world, [tuple(range(1, world))], backend="nccl", timeout=600)


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
