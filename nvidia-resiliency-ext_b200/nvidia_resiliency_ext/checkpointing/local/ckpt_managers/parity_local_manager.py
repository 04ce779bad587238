"""``ParityLocalCheckpointManager``: erasure-coded local checkpoints -- XOR or Reed-Solomon parity per clique member (opt-in).

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

``parity_count = m >= 2`` (Reed-Solomon over GF(2^8), ``b200/erasure.py``): every member cuts its image into ``k = F-m``
fragments, every member holds m parity fragments (rows p of the stripes it holds), and any m lost members of a clique
are rebuilt.  Each rank stores its own file plus ``iter_<it>_<r>_local.rs<m>of<F>.pt`` with its m parity fragments:
``S + m·S/(F-m)`` per rank.  The save runs m pack passes (pass p stores each fragment at the row-p holder of its
stripe), then ONE ``nvrx_gf_combine`` of the ``m·k`` exchange slots into the m parity rows.  ``m = 1`` is the XOR layout
above, with ``nvrx_xor_reduce``.
"""

from __future__ import annotations

import logging
import pickle
import re
from collections import defaultdict
from typing import List, Tuple

import numpy as np
import torch
import torch.distributed as dist

from ...b200 import erasure, fastsave
from ...utils import debug_time
from ..replication.group_utils import GroupWrapper, parse_group_sequence
from .base_manager import CheckpointingException
from .sharded_local_manager import _ALIGN, ShardedLocalCheckpointManager, shard_bytes_for

logger = logging.getLogger(__name__)

ParityID = Tuple[int, int, int]  # (iteration, holder rank, clique size F)
_MAX_PARITY = 4  # destinations of one nvrx_gf_combine


class ParityLocalCheckpointManager(ShardedLocalCheckpointManager):
    """See module docstring.  Constructor and :meth:`from_replication_params` as for ``ShardedLocalCheckpointManager``
    (a clique needs at least 2 members) plus ``parity_count`` (m, ``1 <= m <= min(F-1, 4)``, default 1: XOR parity, one
    loss per clique); ``save / find_latest / load`` as for ``LocalCheckpointManager``."""

    def __init__(self, root_local_ckpt_dir, session_id: str = "", *, clique, parity_count: int = 1):
        super().__init__(root_local_ckpt_dir, session_id, clique=clique)
        F = len(self._members)
        if not 1 <= parity_count <= min(F - 1, _MAX_PARITY):
            raise ValueError(f"parity_count must be between 1 and min(F-1, {_MAX_PARITY}) = {min(F - 1, _MAX_PARITY)}, got {parity_count}")
        if parity_count > 1 and parity_count * (F - parity_count) > 64:
            raise ValueError(f"parity_count {parity_count} at F = {F}: a holder combines m·(F-m) > 64 fragments")
        self._m = parity_count
        self._code = erasure.StripeLayout(self._members, parity_count)

    @classmethod
    def from_replication_params(cls, root_local_ckpt_dir, session_id: str = "", replication_jump: int = 1,
                                replication_factor: int = 2, parity_count: int = 1) -> "ParityLocalCheckpointManager":
        """Cliques as in ``ShardedLocalCheckpointManager.from_replication_params`` (collective)."""
        cliques = parse_group_sequence(replication_jump, replication_factor, dist.get_world_size())
        groups = [dist.new_group(list(c)) for c in cliques]
        return cls(root_local_ckpt_dir, session_id, clique=GroupWrapper.from_list_of_groups(groups), parity_count=parity_count)

    # ---- naming -------------------------------------------------------------------------------
    def _parity_suffix(self, F) -> str:
        """``.parity<F-1>`` for XOR parity, ``.rs<m>of<F>`` for m >= 2 parity fragments."""
        return f".parity{F - 1}" if self._m == 1 else f".rs{self._m}of{F}"

    def _parity_path(self, pid: ParityID, is_dirty=False):
        it, holder, F = pid
        return self.local_ckpt_dir / self._filename_from_template(it, holder, self._parity_suffix(F) + (".dirty" if is_dirty else ""))

    def _my_parity_ids(self) -> List[ParityID]:
        """Parity files written with this manager's m (files of another m do not count)."""
        self._ensure_dir()
        tag = r"parity(\d+)" if self._m == 1 else rf"rs{self._m}of(\d+)"
        pat = re.compile(rf"iter_(\d+)_(\d+)_local\.{tag}\.pt")
        out = []
        for entry in self.local_ckpt_dir.iterdir():
            m = pat.fullmatch(entry.name)
            if m and entry.is_file():
                it, holder, x = (int(g) for g in m.groups())
                out.append((it, holder, x + 1 if self._m == 1 else x))
        return out

    # ---- coverage -----------------------------------------------------------------------------
    @debug_time("ParityLocalCheckpointManager.find_latest", logger)
    def find_latest(self):
        """Newest iteration at which, in every clique, at most m members lack their own file and every other member has its
        own file and its parity file of that iteration (written with this m and clique size F).  Collective."""
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
            for it, holder, F in pids:
                have_parity[it].add((holder, F))
        cliques = {g[2] for g in gathered}

        def complete(it):
            for clique in cliques:
                missing = [m for m in clique if m not in have_full[it]]
                if len(missing) > self._m:
                    return False
                if any((m, len(clique)) not in have_parity[it] for m in clique if m not in missing):
                    return False
            return True

        self.latest_iteration = max((it for it in set(have_full) | set(have_parity) if complete(it)), default=-1)
        return self.latest_iteration

    # ---- save -----------------------------------------------------------------------------------
    def _save_fragment(self, spec: dict):
        """Writer side: the parity file of this holder (``.dirty`` name, renamed when complete)."""
        self._ensure_dir()
        pid = (spec["iteration"], spec["holder"], len(spec["members"]))
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
        spec = {"iteration": iteration, "holder": me, "n": len(self._members) - 1, "members": list(self._members),
                "shard_bytes": sb, "senders": senders, "data": data}
        if self._m > 1:
            code = self._code
            spec.update({"parity_count": self._m, "generator": code.G.copy(),
                         "contributors": {s: code.contributors(s) for s in code.held_stripes(me)}})
        return spec

    def _gather_metas(self, my_id, total: int, skeleton_blob, layout) -> Tuple[list, int]:
        """Every member's description and the clique-wide fragment size (from the largest packed image)."""
        metas = self.clique.all_gather_object({"id": my_id, "total": total, "skeleton": skeleton_blob, "layout": layout})
        return metas, shard_bytes_for(max(m["total"] for m in metas), self._code.k)

    def _round(self, row: int, sb: int) -> Tuple[List[int], List[int], int]:
        """Save round ``row`` of the NCCL / gloo exchange: (send splits, receive splits, rotation).  Each fragment goes to
        the row-``row`` holder of its stripe, one fragment per member at most.  Sorted by stripe, the destinations are in
        clique order up to a rotation: the send buffer is the packed image rotated by ``rotation`` fragments."""
        code, me = self._code, self.rank
        dests = [h for h, _ in code.fragment_destinations(me, row)]
        send = [sb if m in dests else 0 for m in self._members]
        senders = code.contributors(code.held_stripes(me)[row])
        recv = [sb if m in senders else 0 for m in self._members]
        order = sorted(range(len(dests)), key=lambda q: self._members.index(dests[q]))
        return send, recv, order[0]

    def _round_send(self, flat: torch.Tensor, rot: int, sb: int) -> torch.Tensor:
        k = self._code.k
        return flat[: k * sb] if rot == 0 else torch.cat([flat[rot * sb : k * sb], flat[: rot * sb]])

    def _encode_host(self, recv: torch.Tensor, sb: int) -> torch.Tensor:
        k = self._code.k
        if self._m == 1:
            return _xor_host([recv[q * sb : (q + 1) * sb] for q in range(k)])
        raw = recv.numpy()
        rows = erasure.combine(self._code.encode_matrix(), [raw[t * sb : (t + 1) * sb] for t in range(self._m * k)])
        return torch.from_numpy(np.concatenate(rows))

    def _exchange_host(self, payload, my_id, skeleton_blob):
        from ...b200.engine import expected_layout

        k = self._code.k
        nbytes = [t.numel() * t.element_size() for t in payload]
        offs, _, total = expected_layout(nbytes, [False] * len(nbytes), _ALIGN)
        layout = {"shapes": [tuple(t.shape) for t in payload], "dtypes": [t.dtype for t in payload], "offsets": offs, "nbytes": nbytes}
        metas, sb = self._gather_metas(my_id, total, skeleton_blob, layout)
        flat = torch.zeros(k * sb, dtype=torch.uint8)  # gaps and the padding past `total` combine as zero
        for t, off, nb in zip(payload, offs, nbytes):
            if nb:
                flat[off : off + nb] = t.detach().contiguous().view(-1).view(torch.uint8)
        recv = torch.empty(self._m * k * sb, dtype=torch.uint8)
        for p in range(self._m):
            send_splits, recv_splits, rot = self._round(p, sb)
            dist.all_to_all_single(recv[p * k * sb : (p + 1) * k * sb], self._round_send(flat, rot, sb), recv_splits, send_splits,
                                   group=self.clique.group)
        parity = self._encode_host(recv, sb)
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
        code = self._code
        k, mp = code.k, self._m
        layout = {"shapes": [tuple(t.shape) for t in payload], "dtypes": [t.dtype for t in payload],
                  "offsets": list(plan.offsets), "nbytes": list(plan.packed_nbytes)}
        metas, sb = self._gather_metas(my_id, total, skeleton_blob, layout)
        me = self.rank
        stream = engine._current_stream()
        xbuf, bases = xch.shared_exchange(engine, self.clique, mp * k * sb)
        free_ev = getattr(engine, "_exchange_free", None)
        if free_ev is not None:
            stream_wait_event(stream, free_ev)
        if bases is not None:
            staging = engine._ensure_staging(total)
            if engine._staging_free is not None:
                stream_wait_event(stream, engine._staging_free)
            if getattr(engine, "_exchange_dirty", True):  # another exchange left bytes in it: peers' gaps must land on zeros
                xch.as_uint8_tensor(xbuf.ptr, xbuf.nbytes, engine.device).zero_()
            plan.set_shard_rotation(code.first_fragment(me))
            xch._clique_barrier(engine, self.clique)
            for p in range(mp):  # pass p: fragment q -> the row-p holder of its stripe; only pass 0 keeps the own copy
                dest = [bases[self._members.index(h)] + slot * sb for h, slot in code.fragment_destinations(me, p)]
                plan.pack_sharded(staging.ptr if p == 0 else None, dest, sb, 0, stream)
                engine.launches += 1 if plan.n_tiles else 0
            xch._clique_barrier(engine, self.clique)
            engine.last_exchange = "p2p-fused-parity"
        else:
            staging = engine._ensure_staging(k * sb)
            if engine._staging_free is not None:
                stream_wait_event(stream, engine._staging_free)
            # all_to_all_single sends staging ranges, gaps and padding included
            xch.as_uint8_tensor(staging.ptr, k * sb, engine.device).zero_()
            plan.pack(staging.ptr, stream)
            engine.launches += 1 if plan.n_tiles else 0
            flat = xch.as_uint8_tensor(staging.ptr, k * sb, engine.device)
            for p in range(mp):
                send_splits, recv_splits, rot = self._round(p, sb)
                recv = xch.as_uint8_tensor(xbuf.ptr + p * k * sb, k * sb, engine.device)
                dist.all_to_all_single(recv, self._round_send(flat, rot, sb), recv_splits, send_splits, group=self.clique.group)
            engine.last_exchange = "nccl-alltoall-parity"

        # off the training stream: reduce / combine (clearing the slots for the next save), then the two drains
        packed_ev = Event(engine.device)
        packed_ev.record(stream)
        side = engine._side
        side.wait_event(packed_ev)
        pbytes = mp * sb
        pbuf = getattr(engine, "_parity_buf", None)
        if pbuf is None or pbuf.nbytes < pbytes:
            if pbuf is not None:
                side.synchronize()  # its last drain is over
                pbuf.close()
            pbuf = engine._parity_buf = DeviceBuffer(pbytes, engine.device)
        slots = [xbuf.ptr + t * sb for t in range(mp * k)]
        if mp == 1:
            xch.xor_reduce(engine, pbuf.ptr, slots, sb, True, side.handle)
        else:
            xch.gf_combine(engine, [pbuf.ptr + p * sb for p in range(mp)], slots, code.encode_matrix(), sb, True, side.handle)
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

        slot_b = engine._acquire_slot(pbytes)
        base = slot_b.drained_total
        check(engine.lib.nvrx_drain(slot_b.buf.data_ptr, pbuf.ptr, pbytes, engine.drain_chunk, slot_b.buf.progress_ptr, base,
                                    side.handle, slot_b.done_event.handle), "nvrx_drain")
        slot_b.drained_total = base + pbytes
        lay_b = PackedLayout(shapes=[(pbytes,)], dtypes=["uint8"], src_dtypes=["uint8"], offsets=[0], packed_nbytes=[pbytes], total_bytes=pbytes)
        snaps.append(Snapshot(engine=engine, slot=slot_b, layout=lay_b, progress_target=slot_b.drained_total, n_total=1))
        parity = slot_b.buf.segment(0, pbytes, torch.uint8, (pbytes,))
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
        if len(lost) > self._m:
            raise CheckpointingException(f"Members {lost} of one clique lost iteration {it}: parity rebuilds at most {self._m}")
        if lost:
            got = self._rebuild_from_parity(it, lost, result)
            if self.rank in lost:
                result = got
        assert result is not None
        return result, ckpt_id

    def _rebuild_from_parity(self, iteration: int, lost: List[int], mine):
        """Collective over the clique (``erasure.StripeLayout.rebuild_plan``): survivors re-pack their images, ONE
        all-to-all brings every collector the parity rows and data fragments it decodes from, each collector decodes its
        stripes (one reduce or combine per stripe) and sends every recovered fragment to its owner; the lost members
        scatter their images."""
        me = self.rank
        code = self._code
        k = code.k
        F = len(self._members)
        on_gpu = self.clique._payload_on_gpu()
        survivors = [m for m in self._members if m not in lost]
        steps = code.rebuild_plan(lost)
        moves = code.transfers(steps)
        engine = staging = None
        if on_gpu:
            from ...b200 import exchange as xch
            from ...b200.engine import SnapshotEngine

            engine = SnapshotEngine.get()
            dev = torch.device("cuda", engine.device)
            torch.cuda.current_stream(engine.device).synchronize()  # the load's restore is done with staging
            if engine._staging_free is not None:
                engine._staging_free.synchronize()
        if me not in lost:
            spec = torch.load(self._parity_path((iteration, me, F)), weights_only=False)
            sb = spec["shard_bytes"]
            if me == survivors[0]:
                for u in lost:
                    self.clique.send_object(spec["senders"][u], u)
            tensors = [t.detach().contiguous() for t in mine.tensors]
            if on_gpu:
                plan = engine._plan_for(tensors, [False] * len(tensors))
                staging = engine._ensure_staging(k * sb)
                flat = xch.as_uint8_tensor(staging.ptr, k * sb, engine.device)
                flat.zero_()
                plan.pack(staging.ptr, engine._current_stream())
                engine.launches += 1 if plan.n_tiles else 0
            else:
                from ...b200.engine import expected_layout

                nbytes = [t.numel() * t.element_size() for t in tensors]
                offs, _, _ = expected_layout(nbytes, [False] * len(nbytes), _ALIGN)
                flat = torch.zeros(k * sb, dtype=torch.uint8)
                for t, off, nb in zip(tensors, offs, nbytes):
                    if nb:
                        flat[off : off + nb] = t.view(-1).view(torch.uint8)
            parity = spec["data"].to(flat.device)

            def piece(src):
                _, kind, idx = src
                return (parity if kind == "parity" else flat)[idx * sb : (idx + 1) * sb]

            # what travels, per peer in clique order, each peer's pieces in plan order
            frags, send_splits, recv_splits, recv_at, cur = [], [], [], {}, 0
            for m in self._members:
                out = moves.get((me, m), []) if m != me else []
                frags += [piece(steps[t].sources[i]) for t, i in out]
                send_splits.append(len(out) * sb)
                inc = moves.get((m, me), []) if m != me else []
                for t, i in inc:
                    recv_at[(t, i)] = cur
                    cur += sb
                recv_splits.append(len(inc) * sb)
            send = torch.cat(frags) if frags else flat[:0]
            recv = torch.empty(cur, dtype=torch.uint8, device=flat.device)
            if len(survivors) > 1:
                dist.all_to_all_single(recv, send, recv_splits, send_splits, group=self.clique.group)
            for t, step in enumerate(steps):
                if step.collector != me:
                    continue
                srcs = [piece(src) if src[0] == me else recv[recv_at[(t, i)] : recv_at[(t, i)] + sb] for i, src in enumerate(step.sources)]
                nl = len(step.lost)
                if on_gpu:
                    out = torch.empty(nl * sb, dtype=torch.uint8, device=dev)
                    if self._m == 1:
                        xch.xor_reduce(engine, out.data_ptr(), [x.data_ptr() for x in srcs], sb, False, engine._current_stream())
                    else:
                        xch.gf_combine(engine, [out.data_ptr() + d * sb for d in range(nl)], [x.data_ptr() for x in srcs],
                                       step.matrix, sb, False, engine._current_stream())
                elif self._m == 1:
                    out = _xor_host(srcs)
                else:
                    out = torch.from_numpy(np.concatenate(erasure.combine(step.matrix, [x.numpy() for x in srcs])))
                for d, (owner, _) in enumerate(step.lost):
                    self.clique.send_tensor(out[d * sb : (d + 1) * sb], owner)
            return None
        meta = self.clique.recv_object(survivors[0])
        sb, total, layout = meta["shard_bytes"], meta["total_bytes"], meta["layout"]
        if len(survivors) > 1:  # nothing to or from a lost member
            empty = torch.empty(0, dtype=torch.uint8, device=dev if on_gpu else "cpu")
            dist.all_to_all_single(empty, empty, [0] * len(self._members), [0] * len(self._members), group=self.clique.group)
        if on_gpu:
            staging = engine._ensure_staging(k * sb)
            whole = xch.as_uint8_tensor(staging.ptr, k * sb, engine.device)
        else:
            whole = torch.zeros(k * sb, dtype=torch.uint8)
        collector = {(owner, q): step.collector for step in steps for owner, q in step.lost}
        for q in range(k):
            self.clique.recv_tensor(whole[q * sb : (q + 1) * sb], collector[(me, q)])
        return self._scatter_image(pickle.loads(meta["skeleton"]), layout, total, whole, staging)


def _xor_host(parts: List[torch.Tensor]) -> torch.Tensor:
    out = parts[0].clone()
    for p in parts[1:]:
        torch.bitwise_xor(out, p, out=out)
    return out
