"""ParityLocalCheckpointManager host logic on gloo (world sizes 3, 4, 6 and 8): one XOR parity fragment per member, the
coverage rule, rebuild of one lost member per clique, fallback when two members of a clique are lost, cleanup."""
import numpy as np
import pytest
import torch
import torch.distributed as dist

from _mp import run_ranks


def make_sd(seed):
    g = torch.Generator().manual_seed(seed)
    # sizes differ per rank: images of different lengths, gaps between the tensors
    return {"w": torch.randn(301 + 53 * (seed % 7), 9, generator=g), "opt": [{"m": torch.randn(33, generator=g).to(torch.bfloat16), "step": torch.tensor(float(seed))}],
            "ids": torch.randint(0, 10, (5 + seed % 3,), generator=g), "note": f"seed{seed}", "empty": torch.empty(0, 2)}


def same(a, b):
    ta, tb = list(a.tensors), list(b.tensors)
    return len(ta) == len(tb) and all(x.dtype == y.dtype and x.shape == y.shape and torch.equal(x.cpu(), y.cpu()) for x, y in zip(ta, tb)) and a.state_dict["note"] == b.state_dict["note"]


def packed_image(sd, length):
    """The dense packed image of a state dict's tensors, zero-padded to ``length`` bytes (the layout rule of the engine)."""
    from _cpu_tasd import CpuTensorAwareStateDict
    from nvidia_resiliency_ext.checkpointing.b200.engine import expected_layout

    tensors = list(CpuTensorAwareStateDict(sd).tensors)
    nbytes = [t.numel() * t.element_size() for t in tensors]
    offs, _, total = expected_layout(nbytes, [False] * len(nbytes), 512)
    img = np.zeros(max(length, total), dtype=np.uint8)
    for t, off, nb in zip(tensors, offs, nbytes):
        img[off : off + nb] = t.contiguous().view(-1).view(torch.uint8).numpy()
    return img, total


def expected_parity(mgr, holder, seed_of):
    """P_holder = XOR over the other members i of fragment ``_others(i).index(holder)`` of i's image."""
    from nvidia_resiliency_ext.checkpointing.local.ckpt_managers.sharded_local_manager import shard_bytes_for

    n = len(mgr._members) - 1
    totals = {m: packed_image(make_sd(seed_of(m)), 0)[1] for m in mgr._members}
    sb = shard_bytes_for(max(totals.values()), n)
    out = np.zeros(sb, dtype=np.uint8)
    for i in mgr._others(holder):
        img, _ = packed_image(make_sd(seed_of(i)), n * sb)
        k = mgr._others(i).index(holder)
        out ^= img[k * sb : (k + 1) * sb]
    return out, sb, totals


def _w(rank, world, root, jump, factor, is_async):
    import time

    from _cpu_tasd import CpuTensorAwareStateDict
    from nvidia_resiliency_ext.checkpointing.async_ckpt.core import AsyncCallsQueue
    from nvidia_resiliency_ext.checkpointing.local.ckpt_managers.parity_local_manager import ParityLocalCheckpointManager

    mgr = ParityLocalCheckpointManager.from_replication_params(root, replication_jump=jump, replication_factor=factor)
    members = mgr._members
    n = len(members) - 1
    q = AsyncCallsQueue(persistent=False)

    def save(it, m=mgr):
        req = m.save(CpuTensorAwareStateDict(make_sd(100 * it + rank)), it, is_async=is_async)
        if is_async:
            q.schedule_async_request(req)
            q.maybe_finalize_async_calls(blocking=True, no_dist=False)
        else:
            assert req is None

    for it in (1, 2):
        save(it)
    time.sleep(0.5)  # async cleanup of iteration 1
    files = sorted(p.name for p in mgr.local_ckpt_dir.iterdir())
    assert files == sorted([f"iter_0000002_{rank}_local.pt", f"iter_0000002_{rank}_local.parity{n}.pt"]), files

    # the parity file: frag_slot bytes equal to the XOR of the peers' fragments, plus what a survivor needs to describe a loss
    spec = torch.load(mgr.local_ckpt_dir / f"iter_0000002_{rank}_local.parity{n}.pt", weights_only=False)
    want, sb, totals = expected_parity(mgr, rank, lambda m: 200 + m)
    assert spec["shard_bytes"] == sb and spec["data"].numel() == sb and spec["data"].dtype == torch.uint8
    assert np.array_equal(spec["data"].numpy(), want)
    assert spec["members"] == members and spec["n"] == n and spec["holder"] == rank
    assert sorted(spec["senders"]) == [m for m in members if m != rank]
    assert all(spec["senders"][m]["total_bytes"] == totals[m] and spec["senders"][m]["shard_bytes"] == sb for m in spec["senders"])
    dist.barrier()

    # one member of every clique loses its storage: rebuilt bit-identically
    lost = members[world % len(members)]  # the same choice on every member of a clique
    if rank == lost:
        for p in mgr.local_ckpt_dir.iterdir():
            p.unlink()
    dist.barrier()
    mgr2 = ParityLocalCheckpointManager(root, clique=mgr.clique)
    assert mgr2.find_latest() == 2
    loaded, cid = mgr2.load()
    assert cid == (2, rank, "") and same(loaded, CpuTensorAwareStateDict(make_sd(200 + rank)))
    dist.barrier()

    # iteration 3 with the cleanup of iteration 2 held back; two members of one clique lose iteration 3: iteration 2 (one
    # loss per clique) is the newest complete one
    mgr3 = ParityLocalCheckpointManager(root, clique=mgr.clique)
    mgr3._cleanup = lambda iteration: None
    save(3, mgr3)
    clique0 = next(c for c in gathered_cliques(mgr) if 0 in c)
    if rank in clique0[:2]:
        for p in mgr.local_ckpt_dir.glob("iter_0000003_*"):
            p.unlink()
    dist.barrier()
    mgr4 = ParityLocalCheckpointManager(root, clique=mgr.clique)
    assert mgr4.find_latest() == 2
    loaded, cid = mgr4.load()
    assert cid == (2, rank, "") and same(loaded, CpuTensorAwareStateDict(make_sd(200 + rank)))
    q.close()


def gathered_cliques(mgr):
    out = [None] * dist.get_world_size()
    dist.all_gather_object(out, tuple(mgr._members))
    return sorted(set(out))


@pytest.mark.parametrize("world,jump,factor,is_async", [
    (3, 1, 3, True), (4, 1, 2, False), (4, 2, 2, True), (4, 1, 4, False),
    (6, 1, 3, True), (6, 2, 3, False), (8, 1, 8, True), (8, 2, 4, False),
])
def test_parity_save_and_rebuild(tmp_path, world, jump, factor, is_async):
    run_ranks(_w, world, str(tmp_path), jump, factor, is_async, timeout=300)


def _w_pair(rank, world, root):
    from _cpu_tasd import CpuTensorAwareStateDict
    from nvidia_resiliency_ext.checkpointing.local.ckpt_managers.parity_local_manager import ParityLocalCheckpointManager
    from nvidia_resiliency_ext.checkpointing.local.ckpt_managers.sharded_local_manager import ShardedLocalCheckpointManager

    par = ParityLocalCheckpointManager.from_replication_params(root + "/parity", replication_jump=1, replication_factor=2)
    striped = ShardedLocalCheckpointManager.from_replication_params(root + "/striped", replication_jump=1, replication_factor=2)
    par.save(CpuTensorAwareStateDict(make_sd(rank)), 1)
    striped.save(CpuTensorAwareStateDict(make_sd(rank)), 1)
    # F = 2: the parity is the one fragment striping would store, zero-padded to the clique's fragment size
    other = par._others(rank)[0]
    p = torch.load(par.local_ckpt_dir / f"iter_0000001_{rank}_local.parity1.pt", weights_only=False)["data"]
    f = torch.load(striped.local_ckpt_dir / f"iter_0000001_{other}_local.s0of1.pt", weights_only=False)["data"]
    assert torch.equal(p[: f.numel()], f) and int(p[f.numel():].count_nonzero()) == 0
    dist.barrier()
    # a parity file still under its .dirty name does not count: the iteration is not complete (a save that left it so fails)
    if rank == 1:
        done = par.local_ckpt_dir / "iter_0000001_1_local.parity1.pt"
        done.rename(par.local_ckpt_dir / "iter_0000001_1_local.parity1.dirty.pt")
    dist.barrier()
    assert ParityLocalCheckpointManager(root + "/parity", clique=par.clique).find_latest() == -1
    # a failed save's cleanup removes complete and dirty files of that iteration, as for the striped manager
    par._cleanup_failed_save(1)
    assert list(par.local_ckpt_dir.iterdir()) == []


def test_parity_pair_equals_striped_fragment_and_dirty_files(tmp_path):
    run_ranks(_w_pair, 2, str(tmp_path))
