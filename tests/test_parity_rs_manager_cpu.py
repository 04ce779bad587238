"""ParityLocalCheckpointManager with parity_count m >= 2 (Reed-Solomon over GF(2^8)) on gloo, world sizes 3 to 8: file
names, parity bytes against an oracle computed from the images, rebuild of every lost set of at most m members of one
clique, fallback after m + 1 losses, files of another m and .dirty files not counted, cleanup, and m = 1 given
explicitly writing what the default writes."""
import itertools

import numpy as np
import pytest
import torch
import torch.distributed as dist

from _mp import run_ranks
from test_parity_manager_cpu import make_sd, packed_image, same


def slow_mul(a, b):
    r = 0
    for _ in range(8):
        if b & 1:
            r ^= a
        b >>= 1
        a <<= 1
        if a & 0x100:
            a ^= 0x11D
    return r


def expected_rs_parity(mgr, holder, seed_of):
    """The m parity rows ``holder`` keeps: row p = sum over the contributors j of its stripe of G[p][j] · their fragment."""
    from nvidia_resiliency_ext.checkpointing.local.ckpt_managers.sharded_local_manager import shard_bytes_for

    code = mgr._code
    totals = {r: packed_image(make_sd(seed_of(r)), 0)[1] for r in mgr._members}
    sb = shard_bytes_for(max(totals.values()), code.k)
    rows = []
    for p, s in enumerate(code.held_stripes(holder)):
        out = np.zeros(sb, dtype=np.uint8)
        for j, c in enumerate(code.contributors(s)):
            img, _ = packed_image(make_sd(seed_of(c)), code.k * sb)
            q = code.stripes_of(c).index(s)
            table = np.array([slow_mul(int(code.G[p, j]), x) for x in range(256)], dtype=np.uint8)
            out ^= table[img[q * sb : (q + 1) * sb]]
        rows.append(out)
    return np.concatenate(rows), sb, totals


def gathered_cliques(mgr):
    out = [None] * dist.get_world_size()
    dist.all_gather_object(out, tuple(mgr._members))
    return sorted(set(out))


def _w(rank, world, root, jump, factor, m, is_async):
    import time

    from _cpu_tasd import CpuTensorAwareStateDict
    from nvidia_resiliency_ext.checkpointing.async_ckpt.core import AsyncCallsQueue
    from nvidia_resiliency_ext.checkpointing.local.ckpt_managers.parity_local_manager import ParityLocalCheckpointManager

    mgr = ParityLocalCheckpointManager.from_replication_params(root, replication_jump=jump, replication_factor=factor, parity_count=m)
    members = mgr._members
    F = len(members)
    q = AsyncCallsQueue(persistent=False)

    def save(it, man=mgr):
        req = man.save(CpuTensorAwareStateDict(make_sd(100 * it + rank)), it, is_async=is_async)
        if is_async:
            q.schedule_async_request(req)
            q.maybe_finalize_async_calls(blocking=True, no_dist=False)
        else:
            assert req is None

    for it in (1, 2):
        save(it)
    time.sleep(0.5)  # async cleanup of iteration 1
    rs = f"iter_0000002_{rank}_local.rs{m}of{F}.pt"
    files = sorted(p.name for p in mgr.local_ckpt_dir.iterdir())
    assert files == sorted([f"iter_0000002_{rank}_local.pt", rs]), files

    spec = torch.load(mgr.local_ckpt_dir / rs, weights_only=False)
    want, sb, totals = expected_rs_parity(mgr, rank, lambda r: 200 + r)
    assert spec["shard_bytes"] == sb and spec["data"].dtype == torch.uint8 and spec["data"].numel() == m * sb
    assert np.array_equal(spec["data"].numpy(), want)
    assert spec["members"] == members and spec["holder"] == rank and spec["parity_count"] == m
    assert np.array_equal(spec["generator"], mgr._code.G)
    assert spec["contributors"] == {s: mgr._code.contributors(s) for s in mgr._code.held_stripes(rank)}
    assert sorted(spec["senders"]) == [r for r in members if r != rank]
    assert all(spec["senders"][r]["total_bytes"] == totals[r] and spec["senders"][r]["shard_bytes"] == sb for r in spec["senders"])
    dist.barrier()

    # every lost set of at most m members of clique 0 (the same sets, by position, in the other cliques); a new save
    # between patterns
    it = 2
    for t in range(1, m + 1):
        for pos in itertools.combinations(range(F), t):
            lost = [members[i] for i in pos]
            if rank in lost:
                for p in mgr.local_ckpt_dir.glob(f"iter_{it:07d}_*"):
                    p.unlink()
            dist.barrier()
            probe = ParityLocalCheckpointManager(root, clique=mgr.clique, parity_count=m)
            assert probe.find_latest() == it
            loaded, cid = probe.load()
            assert cid == (it, rank, "") and same(loaded, CpuTensorAwareStateDict(make_sd(100 * it + rank))), (lost, rank)
            dist.barrier()
            it += 1
            save(it, probe)
            mgr = probe
    time.sleep(0.5)

    # m + 1 losses in clique 0 at iteration `it + 1` (its cleanup held back): iteration `it` is the newest complete one
    held = ParityLocalCheckpointManager(root, clique=mgr.clique, parity_count=m)
    held._cleanup = lambda iteration: None
    save(it + 1, held)
    clique0 = next(c for c in gathered_cliques(mgr) if 0 in c)
    if rank in clique0[: m + 1]:
        for p in mgr.local_ckpt_dir.glob(f"iter_{it + 1:07d}_*"):
            p.unlink()
    dist.barrier()
    fb = ParityLocalCheckpointManager(root, clique=mgr.clique, parity_count=m)
    assert fb.find_latest() == it
    loaded, cid = fb.load()
    assert cid == (it, rank, "") and same(loaded, CpuTensorAwareStateDict(make_sd(100 * it + rank)))
    dist.barrier()
    # a manager with another m counts none of these parity files
    other = 1 if m > 1 else 2
    assert ParityLocalCheckpointManager(root, clique=mgr.clique, parity_count=other).find_latest() == -1
    q.close()


@pytest.mark.parametrize("world,jump,factor,m,is_async", [
    (3, 1, 3, 2, True), (4, 1, 4, 2, False), (4, 1, 4, 3, True), (5, 1, 5, 3, False),
    (6, 2, 3, 2, False), (6, 1, 6, 2, True), (8, 2, 4, 2, True), (8, 1, 8, 3, False),
])
def test_rs_save_rebuild_and_fallback(tmp_path, world, jump, factor, m, is_async):
    run_ranks(_w, world, str(tmp_path), jump, factor, m, is_async, timeout=600)


def _w_files(rank, world, root):
    from _cpu_tasd import CpuTensorAwareStateDict
    from nvidia_resiliency_ext.checkpointing.local.ckpt_managers.parity_local_manager import ParityLocalCheckpointManager

    m = 2
    mgr = ParityLocalCheckpointManager.from_replication_params(root + "/rs", replication_jump=1, replication_factor=world, parity_count=m)
    mgr.save(CpuTensorAwareStateDict(make_sd(rank)), 1)
    rs = mgr.local_ckpt_dir / f"iter_0000001_{rank}_local.rs{m}of{world}.pt"
    assert rs.exists()
    dist.barrier()
    # a parity file still under its .dirty name does not count
    if rank == 1:
        rs.rename(mgr.local_ckpt_dir / f"iter_0000001_1_local.rs{m}of{world}.dirty.pt")
    dist.barrier()
    assert ParityLocalCheckpointManager(root + "/rs", clique=mgr.clique, parity_count=m).find_latest() == -1
    # a failed save's cleanup removes complete and dirty files of that iteration
    mgr._cleanup_failed_save(1)
    assert list(mgr.local_ckpt_dir.iterdir()) == []
    dist.barrier()

    # m = 1 given explicitly: the same names and bytes as the default
    dflt = ParityLocalCheckpointManager.from_replication_params(root + "/d", replication_jump=1, replication_factor=world)
    one = ParityLocalCheckpointManager.from_replication_params(root + "/e", replication_jump=1, replication_factor=world, parity_count=1)
    dflt.save(CpuTensorAwareStateDict(make_sd(rank)), 1)
    one.save(CpuTensorAwareStateDict(make_sd(rank)), 1)
    a = sorted(p.name for p in dflt.local_ckpt_dir.iterdir())
    b = sorted(p.name for p in one.local_ckpt_dir.iterdir())
    assert a == b == sorted([f"iter_0000001_{rank}_local.pt", f"iter_0000001_{rank}_local.parity{world - 1}.pt"])
    for name in a:
        assert (dflt.local_ckpt_dir / name).read_bytes() == (one.local_ckpt_dir / name).read_bytes(), name


def test_rs_dirty_cleanup_and_default_m(tmp_path):
    run_ranks(_w_files, 4, str(tmp_path))


def test_parity_count_bounds(tmp_path):
    run_ranks(_w_bounds, 6, str(tmp_path))


def _w_bounds(rank, world, root):
    from nvidia_resiliency_ext.checkpointing.local.ckpt_managers.parity_local_manager import ParityLocalCheckpointManager

    mgr = ParityLocalCheckpointManager.from_replication_params(root, replication_jump=1, replication_factor=world, parity_count=4)
    assert mgr._code.k == 2
    for bad in (0, 5, 6):
        with pytest.raises(ValueError):
            ParityLocalCheckpointManager(root, clique=mgr.clique, parity_count=bad)
