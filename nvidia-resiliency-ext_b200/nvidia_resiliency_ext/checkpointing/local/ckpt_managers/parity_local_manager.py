"""``ParityLocalCheckpointManager``: erasure-coded local checkpoints -- one XOR parity fragment per clique member (opt-in).

The striped layout (``ShardedLocalCheckpointManager``) makes every rank keep its own snapshot plus one fragment of each of
its ``F-1`` peers: ``2·S`` of host memory and D2H per save.  Here the ``F-1`` fragments a member receives are reduced to
one on the GPU, so every rank stores

    its own full snapshot            ``iter_<it>_<r>_local.pt``            (the same file the other managers write)
    one parity fragment              ``iter_<it>_<r>_local.parity<n>.pt``  ``P_r = XOR over i != r of D_i^r``

(``D_i^r``: the fragment of member i's packed image that striping sends to r, ``n = F-1``): ``S + S/(F-1)`` per rank.
The parity file also holds the clique's member list and, for every sender, its skeleton, layout, ``total_bytes`` and
``shard_bytes``, so any single survivor can describe a lost member.  A lost member j comes back as
``D_j^r = P_r XOR (XOR over i not in {r, j} of D_i^r)`` for every r != j: survivors re-pack their loaded tensors, ONE
all-to-all moves the fragments between survivors, every holder reduces and sends its piece to j, and j scatters the image.

All members of a clique cut their image into fragments of the same ``shard_bytes`` (from the largest image of the clique)
so that fragments of different senders line up byte for byte.  Bytes no tensor covers must XOR as zero, or a rebuild
would carry stale bytes into another member's tensors: the fused path keeps its exchange buffer clear (the reduce zeroes
what it read, and a buffer another exchange used is cleared first), the NCCL path clears the staging it sends, the host
path and the rebuild start from zeros.
"""

from __future__ import annotations

import logging
import pickle
import re
from collections import defaultdict
from typing import List, Tuple

import torch
import torch.distributed as dist

from ...b200 import fastsave
from ...utils import debug_time
from ..replication.group_utils import GroupWrapper
from .base_manager import CheckpointingException
from .sharded_local_manager import _ALIGN, ShardedLocalCheckpointManager, shard_bytes_for

logger = logging.getLogger(__name__)

ParityID = Tuple[int, int, int]  # (iteration, holder rank, fragment count n)


class ParityLocalCheckpointManager(ShardedLocalCheckpointManager):
    """See module docstring.  Constructor and :meth:`from_replication_params` as for ``ShardedLocalCheckpointManager``
    (a clique needs at least 2 members); ``save / find_latest / load`` as for ``LocalCheckpointManager``."""

    # ---- naming -------------------------------------------------------------------------------
    def _parity_path(self, pid: ParityID, is_dirty=False):
        it, holder, n = pid
        return self.local_ckpt_dir / self._filename_from_template(it, holder, f".parity{n}" + (".dirty" if is_dirty else ""))

    def _my_parity_ids(self) -> List[ParityID]:
        self._ensure_dir()
        pat = re.compile(r"iter_(\d+)_(\d+)_local\.parity(\d+)\.pt")
        out = []
        for entry in self.local_ckpt_dir.iterdir():
            m = pat.fullmatch(entry.name)
            if m and entry.is_file():
                out.append(tuple(int(g) for g in m.groups()))
        return out

    # ---- coverage -----------------------------------------------------------------------------
    @debug_time("ParityLocalCheckpointManager.find_latest", logger)
    def find_latest(self):
        """Newest iteration at which, in every clique, at most one member lacks its own file and every other member has its
        own file and its parity file of that iteration (with ``n = F-1``).  Collective."""
        if self.latest_iteration != -1:
            return self.latest_iteration
        world = GroupWrapper()
        full = [cid for cid in self._my_ckpt_ids() if cid[1] == self.rank]
        parity = [pid for pid in self._my_parity_ids() if pid[1] == self.rank]
        gathered = world.all_gather_object((full, parity, tuple(self._members)))
        self.globally_available_ids = [g[0] for g in gathered]
        have_full = defaultdict(set)
        have_parity = defaultdict(set)
        for ids, pids, _ in gathered:
            for it, owner, session in ids:
                assert session == self.session_id
                have_full[it].add(owner)
            for it, holder, n in pids:
                have_parity[it].add((holder, n))
        cliques = {g[2] for g in gathered}

        def complete(it):
            for clique in cliques:
                missing = [m for m in clique if m not in have_full[it]]
                if len(missing) > 1:
                    return False
                if any((m, len(clique) - 1) not in have_parity[it] for m in clique if m not in missing):
                    return False
            return True

        self.latest_iteration = max((it for it in set(have_full) | set(have_parity) if complete(it)), default=-1)
        return self.latest_iteration

    # ---- save -----------------------------------------------------------------------------------
    def _save_fragment(self, spec: dict):
        """Writer side: the parity file of this holder (``.dirty`` name, renamed when complete)."""
        self._ensure_dir()
        pid = (spec["iteration"], spec["holder"], spec["n"])
        dirty = self._parity_path(pid, True)
        with open(dirty, "x+b") as fh:
            fastsave.save(spec, fh)
        dirty.rename(self._parity_path(pid, False))

    def _parity_spec(self, metas, sb: int, data: torch.Tensor, iteration: int) -> dict:
        me = self.rank
        senders = {
            m: {"skeleton": meta["skeleton"], "layout": meta["layout"], "total_bytes": meta["total"], "shard_bytes": sb}
            for m, meta in zip(self._members, metas) if m != me
        }
        return {"iteration": iteration, "holder": me, "n": len(self._members) - 1, "members": list(self._members),
                "shard_bytes": sb, "senders": senders, "data": data}

    def _gather_metas(self, my_id, total: int, skeleton_blob, layout) -> Tuple[list, int]:
        """Every member's description and the clique-wide fragment size (from the largest packed image)."""
        metas = self.clique.all_gather_object({"id": my_id, "total": total, "skeleton": skeleton_blob, "layout": layout})
        return metas, shard_bytes_for(max(m["total"] for m in metas), len(self._members) - 1)

    def _splits(self, sb: int, skip=()) -> List[int]:
        """``sb`` bytes between this rank and every other member not in ``skip`` (all_to_all_single split sizes)."""
        return [0 if m == self.rank or m in skip else sb for m in self._members]

    def _exchange_host(self, payload, my_id, skeleton_blob):
        from ...b200.engine import expected_layout

        n = len(self._members) - 1
        nbytes = [t.numel() * t.element_size() for t in payload]
        offs, _, total = expected_layout(nbytes, [False] * len(nbytes), _ALIGN)
        layout = {"shapes": [tuple(t.shape) for t in payload], "dtypes": [t.dtype for t in payload], "offsets": offs, "nbytes": nbytes}
        metas, sb = self._gather_metas(my_id, total, skeleton_blob, layout)
        flat = torch.zeros(n * sb, dtype=torch.uint8)  # gaps and the padding past `total` XOR as zero
        for t, off, nb in zip(payload, offs, nbytes):
            if nb:
                flat[off : off + nb] = t.detach().contiguous().view(-1).view(torch.uint8)
        recv = torch.empty(n * sb, dtype=torch.uint8)
        splits = self._splits(sb)
        dist.all_to_all_single(recv, flat, splits, splits, group=self.clique.group)
        parity = _xor_host([recv[k * sb : (k + 1) * sb] for k in range(n)])
        raw = flat.numpy()
        own_views = [
            torch.frombuffer(raw[off : off + nb], dtype=t.dtype).view(t.shape) if nb else torch.empty(t.shape, dtype=t.dtype)
            for t, off, nb in zip(payload, offs, nbytes)
        ]
        return own_views, [self._parity_spec(metas, sb, parity, my_id[0])], []

    def _exchange_gpu(self, payload, my_id, skeleton_blob):
        from ...b200 import exchange as xch
        from ...b200._cabi import check
        from ...b200.engine import DeviceBuffer, Event, PackedLayout, Snapshot, SnapshotEngine, dtype_name, host_views, stream_wait_event

        assert all(t.is_cuda for t in payload), "mixed CPU/CUDA payloads are not supported"
        payload = [t if t.is_contiguous() else t.detach().contiguous() for t in payload]
        engine = SnapshotEngine.get(payload[0].device.index)
        plan = engine._plan_for(payload, [False] * len(payload))
        total = plan.staging_bytes
        n = len(self._members) - 1
        layout = {"shapes": [tuple(t.shape) for t in payload], "dtypes": [t.dtype for t in payload],
                  "offsets": list(plan.offsets), "nbytes": list(plan.packed_nbytes)}
        metas, sb = self._gather_metas(my_id, total, skeleton_blob, layout)
        me = self.rank
        stream = engine._current_stream()
        xbuf, bases = xch.shared_exchange(engine, self.clique, n * sb)
        free_ev = getattr(engine, "_exchange_free", None)
        if free_ev is not None:
            stream_wait_event(stream, free_ev)
        if bases is not None:
            staging = engine._ensure_staging(total)
            if engine._staging_free is not None:
                stream_wait_event(stream, engine._staging_free)
            if getattr(engine, "_exchange_dirty", True):  # another exchange left bytes in it: peers' gaps must land on zeros
                xch.as_uint8_tensor(xbuf.ptr, xbuf.nbytes, engine.device).zero_()
            dest = [bases[self._members.index(m)] + self._slot_of_sender(me, m) * sb for m in self._others(me)]
            nxt = self._members[(self._members.index(me) + 1) % len(self._members)]
            plan.set_shard_rotation(self._others(me).index(nxt))
            xch._clique_barrier(engine, self.clique)
            plan.pack_sharded(staging.ptr, dest, sb, 0, stream)
            engine.launches += 1 if plan.n_tiles else 0
            xch._clique_barrier(engine, self.clique)
            engine.last_exchange = "p2p-fused-parity"
        else:
            staging = engine._ensure_staging(n * sb)
            if engine._staging_free is not None:
                stream_wait_event(stream, engine._staging_free)
            # all_to_all_single sends staging ranges, gaps and padding included
            xch.as_uint8_tensor(staging.ptr, n * sb, engine.device).zero_()
            plan.pack(staging.ptr, stream)
            engine.launches += 1 if plan.n_tiles else 0
            splits = self._splits(sb)
            send = xch.as_uint8_tensor(staging.ptr, n * sb, engine.device)
            recv = xch.as_uint8_tensor(xbuf.ptr, n * sb, engine.device)
            dist.all_to_all_single(recv, send, splits, splits, group=self.clique.group)
            engine.last_exchange = "nccl-alltoall-parity"

        # off the training stream: reduce (clearing the slots for the next save), then the two drains
        packed_ev = Event(engine.device)
        packed_ev.record(stream)
        side = engine._side
        side.wait_event(packed_ev)
        pbuf = getattr(engine, "_parity_buf", None)
        if pbuf is None or pbuf.nbytes < sb:
            if pbuf is not None:
                side.synchronize()  # its last drain is over
                pbuf.close()
            pbuf = engine._parity_buf = DeviceBuffer(sb, engine.device)
        xch.xor_reduce(engine, pbuf.ptr, [xbuf.ptr + k * sb for k in range(n)], sb, True, side.handle)
        reduced = Event(engine.device)
        reduced.record(side.handle)
        engine._exchange_free = reduced
        engine._exchange_dirty = False

        snaps = []
        slot_a = engine._acquire_slot(total)
        base = slot_a.drained_total
        check(engine.lib.nvrx_drain(slot_a.buf.data_ptr, staging.ptr, total, engine.drain_chunk, slot_a.buf.progress_ptr, base,
                                    side.handle, slot_a.done_event.handle), "nvrx_drain")
        slot_a.drained_total = base + total
        engine._staging_free = slot_a.done_event
        names = [dtype_name(t.dtype) for t in payload]
        lay_a = PackedLayout(shapes=[tuple(t.shape) for t in payload], dtypes=names, src_dtypes=list(names), offsets=list(plan.offsets),
                             packed_nbytes=list(plan.packed_nbytes), total_bytes=total)
        snaps.append(Snapshot(engine=engine, slot=slot_a, layout=lay_a, progress_target=slot_a.drained_total, n_total=len(payload)))
        own_views = host_views(lay_a, slot_a.buf)

        slot_b = engine._acquire_slot(sb)
        base = slot_b.drained_total
        check(engine.lib.nvrx_drain(slot_b.buf.data_ptr, pbuf.ptr, sb, engine.drain_chunk, slot_b.buf.progress_ptr, base,
                                    side.handle, slot_b.done_event.handle), "nvrx_drain")
        slot_b.drained_total = base + sb
        lay_b = PackedLayout(shapes=[(sb,)], dtypes=["uint8"], src_dtypes=["uint8"], offsets=[0], packed_nbytes=[sb], total_bytes=sb)
        snaps.append(Snapshot(engine=engine, slot=slot_b, layout=lay_b, progress_target=slot_b.drained_total, n_total=1))
        parity = slot_b.buf.segment(0, sb, torch.uint8, (sb,))
        return own_views, [self._parity_spec(metas, sb, parity, my_id[0])], snaps

    # ---- load -----------------------------------------------------------------------------------
    @debug_time("ParityLocalCheckpointManager.load", logger)
    def load(self):
        if self.latest_iteration == -1:
            raise CheckpointingException("The 'find_latest' method must be called before invoking the 'load' function.")
        it = self.latest_iteration
        ckpt_id = self._ckpt_id(it)
        have_own = self._local_ckpt_path_from_id(ckpt_id).exists()
        needs = self.clique.all_gather_object(not have_own)
        result = self._load_fn(ckpt_id) if have_own else None
        lost = [m for m, need in zip(self._members, needs) if need]
        if len(lost) > 1:
            raise CheckpointingException(f"Members {lost} of one clique lost iteration {it}: parity rebuilds one")
        if lost:
            got = self._rebuild_from_parity(it, lost[0], result)
            if lost[0] == self.rank:
                result = got
        assert result is not None
        return result, ckpt_id

    def _rebuild_from_parity(self, iteration: int, lost: int, mine):
        """Collective over the clique: survivors re-pack, exchange fragments, reduce with their parity; ``lost`` scatters."""
        me = self.rank
        n = len(self._members) - 1
        on_gpu = self.clique._payload_on_gpu()
        survivors = [m for m in self._members if m != lost]
        engine = staging = None
        if on_gpu:
            from ...b200 import exchange as xch
            from ...b200.engine import SnapshotEngine

            engine = SnapshotEngine.get()
            dev = torch.device("cuda", engine.device)
            torch.cuda.current_stream(engine.device).synchronize()  # the load's restore is done with staging
            if engine._staging_free is not None:
                engine._staging_free.synchronize()
        if me != lost:
            spec = torch.load(self._parity_path((iteration, me, n)), weights_only=False)
            sb = spec["shard_bytes"]
            if me == self._fragment_holder(lost, 0):
                self.clique.send_object(spec["senders"][lost], lost)
            tensors = [t.detach().contiguous() for t in mine.tensors]
            if on_gpu:
                plan = engine._plan_for(tensors, [False] * len(tensors))
                staging = engine._ensure_staging(n * sb)
                flat = xch.as_uint8_tensor(staging.ptr, n * sb, engine.device)
                flat.zero_()
                plan.pack(staging.ptr, engine._current_stream())
                engine.launches += 1 if plan.n_tiles else 0
            else:
                from ...b200.engine import expected_layout

                nbytes = [t.numel() * t.element_size() for t in tensors]
                offs, _, _ = expected_layout(nbytes, [False] * len(nbytes), _ALIGN)
                flat = torch.zeros(n * sb, dtype=torch.uint8)
                for t, off, nb in zip(tensors, offs, nbytes):
                    if nb:
                        flat[off : off + nb] = t.view(-1).view(torch.uint8)
            # fragment k of my image goes to the k-th other member, except to the lost one
            frags = [flat[k * sb : (k + 1) * sb] for k, m in enumerate(self._others(me)) if m != lost]
            send = torch.cat(frags) if frags else flat[:0]
            splits = self._splits(sb, skip=(lost,))
            recv = torch.empty(sum(splits), dtype=torch.uint8, device=flat.device)
            if len(survivors) > 1:
                dist.all_to_all_single(recv, send, splits, splits, group=self.clique.group)
            parity = spec["data"].to(flat.device)
            srcs = [parity] + [recv[k * sb : (k + 1) * sb] for k in range(len(survivors) - 1)]
            if on_gpu:
                piece = torch.empty(sb, dtype=torch.uint8, device=dev)
                xch.xor_reduce(engine, piece.data_ptr(), [s.data_ptr() for s in srcs], sb, False, engine._current_stream())
            else:
                piece = _xor_host(srcs)
            dist.send(piece, lost, group=self.clique.group)
            return None
        meta = self.clique.recv_object(self._fragment_holder(lost, 0))
        sb, total, layout = meta["shard_bytes"], meta["total_bytes"], meta["layout"]
        if len(survivors) > 1:  # nothing to or from the lost member
            empty = torch.empty(0, dtype=torch.uint8, device=dev if on_gpu else "cpu")
            dist.all_to_all_single(empty, empty, [0] * len(self._members), [0] * len(self._members), group=self.clique.group)
        if on_gpu:
            staging = engine._ensure_staging(n * sb)
            whole = xch.as_uint8_tensor(staging.ptr, n * sb, engine.device)
        else:
            whole = torch.zeros(n * sb, dtype=torch.uint8)
        for k in range(n):
            dist.recv(whole[k * sb : (k + 1) * sb], self._fragment_holder(lost, k), group=self.clique.group)
        return self._scatter_image(pickle.loads(meta["skeleton"]), layout, total, whole, staging)


def _xor_host(parts: List[torch.Tensor]) -> torch.Tensor:
    out = parts[0].clone()
    for p in parts[1:]:
        torch.bitwise_xor(out, p, out=out)
    return out
