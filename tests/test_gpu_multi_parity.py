"""ParityLocalCheckpointManager on >= 2 GPUs (NCCL), one GPU per rank: saves over the fused P2P path and over NCCL, and at
F = 2 the parity equal to the striped fragment.  ``_w_parity`` is shared with ``test_gpu_multi_parity_rs`` and with the
one-device cliques of ``test_gpu_one_device_cliques``: every save's parity and own file against a host computation (with a
shrinking image, after a striped save, and with stale bytes planted in the exchange buffer and staging), one launch per
pack pass plus one combine per save, and rebuilds of lost members bit-exactly."""
import itertools

import numpy as np
import pytest
import torch
import torch.distributed as dist

from _mp import run_ranks
from test_gpu_multi import _image, bit_equal, edge_state, fill_staging, flat_tensors, rank_state
from test_parity_rs_manager_cpu import slow_mul

pytestmark = [pytest.mark.gpu, pytest.mark.multigpu]


def expected_parity(code, holder, images, sb):
    """The parity rows ``holder`` keeps, from the members' packed images (padded to ``k·sb``): row p = sum over the
    contributors j of its stripe of G[p][j] · their fragment, multiplied by shift-and-reduce tables."""
    rows = []
    for p, s in enumerate(code.held_stripes(holder)):
        out = np.zeros(sb, dtype=np.uint8)
        for j, c in enumerate(code.contributors(s)):
            q = code.stripes_of(c).index(s)
            table = np.array([slow_mul(int(code.G[p, j]), x) for x in range(256)], dtype=np.uint8)
            out ^= table[images[c][q * sb : (q + 1) * sb]]
        rows.append(out)
    return np.concatenate(rows)


def walk_start(plan, sb, first):
    """(fragment the fused pack's tile walk starts in, the one it should start in): the first fragment at or after
    ``first`` (cyclically, mod the plan's fragment count) that has tiles.  The rotation changes no byte, only which holder
    every member stores into at a given moment."""
    nb, tiles = plan.tiles(sb)
    pos = [plan.offsets[s] + o for s, _, o in (tiles[:nb] or tiles)]
    n = -(-plan.staging_bytes // sb)
    if n < 2:
        return 0, 0
    present = {x // sb for x in pos}
    return pos[0] // sb, next(f for f in ((first + i) % n for i in range(n)) if f in present)


def lost_sets(members, m, positions):
    """Lost member sets: ``positions`` (indices into the clique), or every set of at most m members when None."""
    if positions is None:
        positions = [pos for t in range(1, m + 1) for pos in itertools.combinations(range(len(members)), t)]
    return [[members[i] for i in pos] for pos in positions]


def _w_parity(rank, world, root, mode, jump, factor, m, positions):
    """Saves of ParityLocalCheckpointManager(parity_count=m) on the device path, parity and own files checked byte for
    byte after every save, then a rebuild of every lost set in ``positions`` (see ``lost_sets``; the same positions in
    every clique) with a new save between them."""
    import os
    import time

    os.environ["NVRX_B200_EXCHANGE"] = mode
    from nvidia_resiliency_ext.checkpointing.async_ckpt.core import AsyncCallsQueue
    from nvidia_resiliency_ext.checkpointing.b200 import exchange as xch
    from nvidia_resiliency_ext.checkpointing.b200.engine import SnapshotEngine
    from nvidia_resiliency_ext.checkpointing.local.basic_state_dict import BasicTensorAwareStateDict
    from nvidia_resiliency_ext.checkpointing.local.ckpt_managers.parity_local_manager import ParityLocalCheckpointManager
    from nvidia_resiliency_ext.checkpointing.local.ckpt_managers.sharded_local_manager import ShardedLocalCheckpointManager, shard_bytes_for

    mgr = ParityLocalCheckpointManager.from_replication_params(root, replication_jump=jump, replication_factor=factor, parity_count=m)
    code, members = mgr._code, mgr._members
    F = len(members)
    suffix = f"parity{F - 1}" if m == 1 else f"rs{m}of{F}"
    branch = "nccl-alltoall-parity" if mode == "nccl" else "p2p-fused-parity"
    q = AsyncCallsQueue(persistent=False)
    engine = SnapshotEngine.get()
    shrunk, plans = {}, {}

    def save(man, it, shrink=False):
        shrunk[it] = shrink
        sd = BasicTensorAwareStateDict(edge_state(10 * it + rank, shrink))
        live = list(sd.tensors)
        launches0 = engine.launches
        req = man.save(sd, it, is_async=True)
        assert engine.last_exchange == branch, engine.last_exchange
        # fused: m pack passes + one combine; collective: one pack + one combine
        assert engine.launches - launches0 == (1 if mode == "nccl" else m) + 1, ("launches", engine.launches - launches0)
        plans[it] = engine._plan_for(live, [False] * len(live))
        q.schedule_async_request(req)
        for t in live:
            t.zero_()  # training goes on: the files must hold the state from before
        assert len(q.maybe_finalize_async_calls(blocking=True, no_dist=False)) == 1

    def want(r, it):
        return flat_tensors(edge_state(10 * it + r, shrunk[it]))

    def check(it):
        states = {r: want(r, it) for r in members}
        own = torch.load(mgr.local_ckpt_dir / f"iter_{it:07d}_{rank}_local.pt", weights_only=False)
        got = list(own.tensors)
        assert len(got) == len(states[rank]) and all(bit_equal(a, b) for a, b in zip(got, states[rank])), ("own file", it)
        totals = {r: _image(states[r], 0)[1] for r in members}
        sb = shard_bytes_for(max(totals.values()), code.k)
        images = {r: _image(states[r], code.k * sb)[0] for r in members}
        spec = torch.load(mgr.local_ckpt_dir / f"iter_{it:07d}_{rank}_local.{suffix}.pt", weights_only=False)
        assert spec["shard_bytes"] == sb and spec["members"] == members and spec["holder"] == rank, ("parity header", it)
        assert spec["data"].dtype == torch.uint8 and spec["data"].numel() == m * sb, ("parity size", it)
        got_p, want_p = spec["data"].numpy(), expected_parity(code, rank, images, sb)
        bad = np.flatnonzero(got_p != want_p)
        assert bad.size == 0, ("parity bytes", it, bad.size, "differ, zero in the file:", int((got_p[bad] == 0).sum()), bad[:8])
        if mode != "nccl":
            start, first = walk_start(plans[it], sb, code.first_fragment(rank))
            assert start == first, ("walk start", it, start, first)
        assert sorted(spec["senders"]) == [r for r in members if r != rank]
        assert all(spec["senders"][r]["total_bytes"] == totals[r] and spec["senders"][r]["shard_bytes"] == sb for r in spec["senders"])
        if m > 1:
            assert spec["parity_count"] == m and np.array_equal(spec["generator"], code.G)
            assert spec["contributors"] == {s: code.contributors(s) for s in code.held_stripes(rank)}

    save(mgr, 1)
    check(1)
    # zero invariant (a): a smaller image than the last save's, nothing planted -- its padding and gaps lie where save 1
    # left bytes, which only the clearing combine removed
    save(mgr, 2, shrink=True)
    check(2)
    # (b): a striped save through the same engine and clique leaves its fragments in the exchange buffer
    striped = ShardedLocalCheckpointManager(root + "/striped", clique=mgr.clique)
    striped.save(BasicTensorAwareStateDict(edge_state(7 + rank)), 1)
    assert engine.last_exchange == ("nccl-alltoall" if mode == "nccl" else "p2p-fused-sharded")
    assert engine._exchange_dirty
    save(mgr, 3, shrink=True)
    check(3)
    # (c): stale bytes planted in the exchange buffer (as another exchange leaves it) and in staging
    xch.as_uint8_tensor(engine._exchange_buf.ptr, engine._exchange_buf.nbytes, engine.device).fill_(0xAB)
    engine._exchange_dirty = True
    fill_staging(engine, 0xCD)
    save(mgr, 4)
    check(4)
    time.sleep(0.5)  # async cleanup of the older iterations
    files = sorted(p.name for p in mgr.local_ckpt_dir.iterdir())
    assert files == sorted([f"iter_0000004_{rank}_local.pt", f"iter_0000004_{rank}_local.{suffix}.pt"]), files
    dist.barrier()

    it = 4
    for lost in lost_sets(members, m, positions):
        if rank in lost:
            for p in mgr.local_ckpt_dir.glob(f"iter_{it:07d}_*"):
                p.unlink()
        dist.barrier()
        fill_staging(engine, 0xCD)  # a re-pack must start from cleared staging
        probe = ParityLocalCheckpointManager(root, clique=mgr.clique, parity_count=m)
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
def test_parity_manager_save_and_rebuild(built_library, shm_dir, mode):
    world = min(torch.cuda.device_count(), 8)
    run_ranks(_w_parity, world, str(shm_dir / mode), mode, 1, world, 1, [(world - 1,)], backend="nccl")


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
