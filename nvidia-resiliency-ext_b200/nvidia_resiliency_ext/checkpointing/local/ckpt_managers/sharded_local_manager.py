"""``ShardedLocalCheckpointManager``: local checkpoints whose replicas are *striped* over the clique (opt-in, new).

The reference replicates by full copies (``CliqueReplicationStrategy``: every member stores every member's shard,
``local/replication/strategies.py:88-140``).  This manager implements the layout of the project's north star instead: the packed
snapshot of rank *r* is cut into ``F-1`` equal fragments, fragment *k* goes to the *k*-th other member of *r*'s clique with
ONE all-to-all over NVLink, and every rank stores

    its own full snapshot            ``iter_<it>_<r>_local.pt``                 (same file the reference would write)
    one fragment of every peer       ``iter_<it>_<owner>_local.s<k>of<n>.pt``   (raw packed bytes + the owner's skeleton)

Host memory and NVLink traffic per rank are ``2·S`` and ``S`` (full replication with factor F needs ``F·S`` and ``(F-1)·S``); any
single member of a clique can lose its storage and gets its snapshot back from the other ``F-1`` members in parallel
(``load``: fragments -> staging -> ONE scatter kernel).  File naming, ``.dirty`` protocol, cleanup and the public methods
(``save / find_latest / load``) are those of ``LocalCheckpointManager``; only the coverage rule is extended: an iteration is
complete when every rank of the world has its full file somewhere **or** all of its fragments are available.

Data path on GPUs of one host: ``nvrx_pack_sharded`` -- ONE kernel reads the tensors once, keeps the full packed copy in the
local staging buffer and stores fragment *k* straight into member *k*'s exchange buffer with NVLink P2P stores (two 4-byte
barriers around it); otherwise pack + ONE ``dist.all_to_all_single`` (NCCL, or gloo for host tensors).
"""

from __future__ import annotations

import logging
from contextlib import nullcontext
import os
import pickle
import re
from collections import defaultdict
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path
from typing import List, Optional, Tuple, Union

import torch
import torch.distributed as dist

from ...async_ckpt.core import AsyncRequest
from ...b200 import fastsave
from ...b200.persist import fast_zip_writes, wait_for_snapshots
from ...utils import _disable_gc, debug_time
from ..base_state_dict import TensorAwareStateDict
from ..replication.group_utils import GroupWrapper, ProcessGroupLike, parse_group_sequence
from .base_manager import CheckpointingException
from .local_manager import LocalCheckpointManager

logger = logging.getLogger(__name__)

_ALIGN = 512
FragID = Tuple[int, int, int, int]  # (iteration, owner rank, fragment index k, fragment count n)


def shard_bytes_for(total_bytes: int, n: int) -> int:
    """Size of one fragment: ``total/n`` rounded up to 512 B (at least 512)."""
    per = -(-total_bytes // max(n, 1))
    return max(_ALIGN, -(-per // _ALIGN) * _ALIGN)


def fragment_range(total_bytes: int, shard_bytes: int, k: int) -> Tuple[int, int]:
    lo = min(total_bytes, k * shard_bytes)
    return lo, min(total_bytes, lo + shard_bytes)


class ShardedLocalCheckpointManager(LocalCheckpointManager):
    """See module docstring.

    Args:
        root_local_ckpt_dir, session_id: as for ``LocalCheckpointManager``.
        clique: the replication group (``ProcessGroup`` / ``GroupWrapper``); build one with
            :meth:`from_replication_params`.  Needs at least 2 members.
    """

    def __init__(self, root_local_ckpt_dir: Union[str, Path], session_id: str = "", *, clique: ProcessGroupLike):
        super().__init__(root_local_ckpt_dir, session_id, repl_strategy=None)
        self.clique: GroupWrapper = GroupWrapper.wrap(clique)
        assert self.clique.world_size >= 2, "striped replication needs at least two clique members"
        self._members: List[int] = list(self.clique.ranks)

    @classmethod
    def from_replication_params(cls, root_local_ckpt_dir, session_id: str = "", replication_jump: int = 1,
                                replication_factor: int = 2) -> "ShardedLocalCheckpointManager":
        """Cliques ``n, n+J, ..., n+(F-1)J`` as in ``CliqueReplicationStrategy.from_replication_params`` (collective)."""
        cliques = parse_group_sequence(replication_jump, replication_factor, dist.get_world_size())
        groups = [dist.new_group(list(c)) for c in cliques]
        return cls(root_local_ckpt_dir, session_id, clique=GroupWrapper.from_list_of_groups(groups))

    # ---- clique geometry ------------------------------------------------------------------------
    def _others(self, member_rank: int) -> List[int]:
        return [m for m in self._members if m != member_rank]

    def _fragment_holder(self, owner: int, k: int) -> int:
        return self._others(owner)[k]

    def _slot_of_sender(self, sender: int, holder: int) -> int:
        """Index of ``sender`` among the members ``holder`` receives fragments from (= holder's exchange slot)."""
        return self._others(holder).index(sender)

    # ---- naming -------------------------------------------------------------------------------
    def _fragment_path(self, frag: FragID, is_dirty=False) -> Path:
        it, owner, k, n = frag
        return self.local_ckpt_dir / self._filename_from_template(it, owner, f".s{k}of{n}" + (".dirty" if is_dirty else ""))

    def _my_fragment_ids(self) -> List[FragID]:
        self._ensure_dir()
        pat = re.compile(r"iter_(\d+)_(\d+)_local\.s(\d+)of(\d+)\.pt")
        out = []
        for entry in self.local_ckpt_dir.iterdir():
            m = pat.fullmatch(entry.name)
            if m and entry.is_file():
                out.append(tuple(int(g) for g in m.groups()))
        return out

    # ---- coverage -----------------------------------------------------------------------------
    @debug_time("ShardedLocalCheckpointManager.find_latest", logger)
    def find_latest(self):
        if self.latest_iteration != -1:
            return self.latest_iteration
        world = GroupWrapper()
        full = [cid for cid in self._my_ckpt_ids() if cid[1] == self.rank]
        frags = self._my_fragment_ids()
        gathered = world.all_gather_object((full, frags))
        self.globally_available_ids = [g[0] for g in gathered]
        self._global_frags = [g[1] for g in gathered]
        have_full = defaultdict(set)
        have_frag = defaultdict(lambda: defaultdict(set))
        for ids, fr in gathered:
            for it, owner, session in ids:
                assert session == self.session_id
                have_full[it].add(owner)
            for it, owner, k, n in fr:
                have_frag[it][(owner, n)].add(k)
        everyone = set(world.ranks)
        best = -1
        for it in set(have_full) | set(have_frag):
            covered = set(have_full[it])
            for (owner, n), ks in have_frag[it].items():
                if len(ks) == n:
                    covered.add(owner)
            if covered >= everyone:
                best = max(best, it)
        self.latest_iteration = best
        return best

    # ---- save -----------------------------------------------------------------------------------
    @debug_time("ShardedLocalCheckpointManager.save", logger)
    def save(self, state_dict: TensorAwareStateDict, iteration: int, is_async: bool = False) -> Optional[AsyncRequest]:
        assert self.latest_iteration < iteration, (
            f"A newer checkpoint is already available: {self.latest_iteration} (saving {iteration})"
        )
        my_id = self._ckpt_id(iteration)
        self._reap_abandoned()  # slots of saves whose queue was aborted (base_manager)
        payload = list(state_dict.pop_tensors())
        skeleton_blob = pickle.dumps(state_dict)  # hollow: a few KB, stored with every fragment
        on_gpu = any(t.is_cuda for t in payload)
        if on_gpu:
            own_views, frag_specs, snaps = self._exchange_gpu(payload, my_id, skeleton_blob)
        else:
            own_views, frag_specs, snaps = self._exchange_host(payload, my_id, skeleton_blob)
        state_dict.insert_tensors(own_views)
        descs = tuple(s.descriptor() for s in snaps)
        self.latest_iteration = -1

        @debug_time("finalize_fn", logger)
        def finalize_fn():
            executor = ThreadPoolExecutor(max_workers=1)
            validated = self.find_latest()
            self.latest_iteration = -1
            for s in snaps:
                s.release()
            if validated < iteration:
                if is_async:
                    executor.submit(self._cleanup_failed_save, iteration)
                    executor.shutdown(wait=False)
                else:
                    self._cleanup_failed_save(iteration)
                raise CheckpointingException(
                    f"Failure during saving local checkpoint from iteration {iteration} (last valid iteration is {validated})"
                )
            if is_async:
                executor.submit(self._cleanup, iteration)
                executor.shutdown(wait=False)
            else:
                self._cleanup(iteration)

        if os.environ.get("NVRX_B200_EAGER_SYNC", "0") not in ("", "0"):
            for s in snaps:
                s.wait()
        args = ({my_id: state_dict}, descs, frag_specs)
        if is_async:
            request = AsyncRequest(self._save_sharded_fn, args, [finalize_fn], async_fn_kwargs={})
            self._track(request, snaps)
            return request
        try:
            self._save_sharded_fn(*args)
        except BaseException:
            for s in snaps:
                s.release()
            raise
        if dist.is_initialized():
            dist.barrier()
        finalize_fn()

    @debug_time("ShardedLocalCheckpointManager._save_sharded_fn", logger)
    @_disable_gc()
    def _save_sharded_fn(self, id_to_state_dict, snapshot_descs, frag_specs):
        """Writer side (forked child or inline): own full file, then one file per received fragment."""
        held = wait_for_snapshots(snapshot_descs)
        try:
            with (fast_zip_writes() if snapshot_descs else nullcontext()), fastsave.slot_ranges(fastsave.ranges_for(snapshot_descs, held)):
                for ckpt_id, sd in id_to_state_dict.items():
                    self._save(sd, ckpt_id)
                for spec in frag_specs:
                    self._save_fragment(spec)
        finally:
            for hb in held:
                hb.close(unlink=False)

    _save_sharded_fn.nvrx_drain_aware = True

    def _save_fragment(self, spec: dict):
        self._ensure_dir()
        frag = (spec["iteration"], spec["owner"], spec["k"], spec["n"])
        dirty = self._fragment_path(frag, True)
        with open(dirty, "x+b") as fh:
            fastsave.save(spec, fh)
        dirty.rename(self._fragment_path(frag, False))

    # ---- exchange: host tensors (CPU backend; host logic / tests) -------------------------------------
    def _exchange_host(self, payload, my_id, skeleton_blob):
        from ...b200.engine import expected_layout

        nbytes = [t.numel() * t.element_size() for t in payload]
        offs, packed, total = expected_layout(nbytes, [False] * len(nbytes), _ALIGN)
        flat = torch.zeros(max(total, 1), dtype=torch.uint8)
        for t, off, nb in zip(payload, offs, nbytes):
            if nb:
                flat[off : off + nb] = t.detach().contiguous().view(-1).view(torch.uint8)
        layout = {"shapes": [tuple(t.shape) for t in payload], "dtypes": [t.dtype for t in payload], "offsets": offs, "nbytes": nbytes}
        metas, recv, in_sizes = self._all_to_all(flat[:total], total, my_id, skeleton_blob, layout)
        raw = flat.numpy()
        own_views = [
            torch.frombuffer(raw[off : off + nb], dtype=t.dtype).view(t.shape) if nb else torch.empty(t.shape, dtype=t.dtype)
            for t, off, nb in zip(payload, offs, nbytes)
        ]
        return own_views, self._fragment_specs(metas, recv, in_sizes, my_id[0]), []

    def _all_to_all(self, send_flat: torch.Tensor, total: int, my_id, skeleton_blob, layout):
        """Metadata all-gather + ONE all_to_all_single of the fragments.  Returns (metas, recv buffer, per-sender sizes)."""
        n = len(self._members) - 1
        sb = shard_bytes_for(total, n)
        metas = self.clique.all_gather_object(
            {"id": my_id, "total": total, "shard_bytes": sb, "skeleton": skeleton_blob, "layout": layout}
        )
        me = self.rank
        in_splits = []  # what I send to each member, in clique order
        for m in self._members:
            if m == me:
                in_splits.append(0)
            else:
                lo, hi = fragment_range(total, sb, self._others(me).index(m))
                in_splits.append(hi - lo)
        out_splits = []  # what each member sends to me
        for m, meta in zip(self._members, metas):
            if m == me:
                out_splits.append(0)
            else:
                lo, hi = fragment_range(meta["total"], meta["shard_bytes"], self._others(m).index(me))
                out_splits.append(hi - lo)
        # fragments of my buffer are contiguous and ordered like _others(me) == clique order without me
        send = send_flat[: sum(in_splits)] if sum(in_splits) else send_flat[:0]
        recv = torch.empty(max(sum(out_splits), 1), dtype=torch.uint8, device=send_flat.device)[: sum(out_splits)]
        dist.all_to_all_single(recv, send.contiguous(), out_splits, in_splits, group=self.clique.group)
        return metas, recv, out_splits

    def _fragment_specs(self, metas, recv_views, sizes, iteration) -> List[dict]:
        """Picklable description of every fragment this rank holds after the exchange (payload = tensor view)."""
        specs, cursor = [], 0
        me = self.rank
        for m, meta, size in zip(self._members, metas, sizes):
            if m == me:
                continue
            # host path: a private copy per fragment (torch.save writes the whole storage a view belongs to)
            data = recv_views[m] if isinstance(recv_views, dict) else recv_views[cursor : cursor + size].clone()
            cursor += size
            specs.append({
                "iteration": iteration, "owner": m, "k": self._others(m).index(me), "n": len(self._members) - 1,
                "shard_bytes": meta["shard_bytes"], "total_bytes": meta["total"], "skeleton": meta["skeleton"],
                "layout": meta["layout"], "data": data,
            })
        return specs

    # ---- exchange: CUDA tensors -----------------------------------------------------------------------
    def _exchange_gpu(self, payload, my_id, skeleton_blob):
        from ...b200 import exchange as xch
        from ...b200.engine import Event, PackedLayout, Snapshot, SnapshotEngine, dtype_name, host_views, stream_wait_event
        from ...b200._cabi import check

        assert all(t.is_cuda for t in payload), "mixed CPU/CUDA payloads are not supported"
        payload = [t if t.is_contiguous() else t.detach().contiguous() for t in payload]
        engine = SnapshotEngine.get(payload[0].device.index)
        plan = engine._plan_for(payload, [False] * len(payload))
        total = plan.staging_bytes
        n = len(self._members) - 1
        sb = shard_bytes_for(total, n)
        layout = {"shapes": [tuple(t.shape) for t in payload], "dtypes": [t.dtype for t in payload],
                  "offsets": list(plan.offsets), "nbytes": list(plan.packed_nbytes)}
        metas = self.clique.all_gather_object(
            {"id": my_id, "total": total, "shard_bytes": sb, "skeleton": skeleton_blob, "layout": layout}
        )
        frag_slot = max(m["shard_bytes"] for m in metas)
        me = self.rank
        stream = engine._current_stream()
        staging = engine._ensure_staging(total)
        xbuf, bases = xch.shared_exchange(engine, self.clique, n * frag_slot)
        if engine._staging_free is not None:
            stream_wait_event(stream, engine._staging_free)
        free_ev = getattr(engine, "_exchange_free", None)
        if free_ev is not None:
            stream_wait_event(stream, free_ev)

        recv_sizes = []
        for m, meta in zip(self._members, metas):
            lo, hi = (0, 0) if m == me else fragment_range(meta["total"], meta["shard_bytes"], self._others(m).index(me))
            recv_sizes.append(hi - lo)
        # If every rank walked its fragments in the same order, all senders would hit the same destination at the same time
        # (incast).  The tile list of a sharded plan interleaves the
        # fragments (destination-major order, csrc/snap_api.cu build_tiles), every GPU stores to all peers at once, and the
        # fused kernel is the default whenever the clique is NVLink-peer reachable; NVRX_B200_EXCHANGE=nccl keeps pack + NCCL.
        if bases is not None:
            # fused: own copy -> staging, fragment k -> member k's exchange buffer (slot = my index among its senders)
            dest = []
            for k, m in enumerate(self._others(me)):
                dest.append(bases[self._members.index(m)] + self._slot_of_sender(me, m) * frag_slot)
            # every member starts its walk at the fragment owned by its right-hand neighbour: distinct destinations
            nxt = self._members[(self._members.index(me) + 1) % len(self._members)]
            plan.set_shard_rotation(self._others(me).index(nxt))
            xch._clique_barrier(engine, self.clique)
            plan.pack_sharded(staging.ptr, dest, sb, 0, stream)
            engine.launches += 1 if plan.n_tiles else 0
            xch._clique_barrier(engine, self.clique)
            engine.last_exchange = "p2p-fused-sharded"
            recv_off = {m: self._others(me).index(m) * frag_slot for m in self._others(me)}
        else:
            plan.pack(staging.ptr, stream)
            engine.launches += 1 if plan.n_tiles else 0
            send = xch.as_uint8_tensor(staging.ptr, total, engine.device)
            in_splits = [0 if m == me else (lambda r: r[1] - r[0])(fragment_range(total, sb, self._others(me).index(m))) for m in self._members]
            recv = xch.as_uint8_tensor(xbuf.ptr, sum(recv_sizes), engine.device)
            dist.all_to_all_single(recv, send[: sum(in_splits)], recv_sizes, in_splits, group=self.clique.group)
            engine.last_exchange = "nccl-alltoall"
            recv_off, cur = {}, 0
            for m, size in zip(self._members, recv_sizes):
                if m != me:
                    recv_off[m] = cur
                    cur += size

        # drains: own packed snapshot -> slot A, received fragments -> slot B
        snaps = []
        packed_ev = Event(engine.device)
        packed_ev.record(stream)
        engine._side.wait_event(packed_ev)
        slot_a = engine._acquire_slot(total)
        base = slot_a.drained_total
        check(engine.lib.nvrx_drain(slot_a.buf.data_ptr, staging.ptr, total, engine.drain_chunk, slot_a.buf.progress_ptr, base,
                                    engine._side.handle, slot_a.done_event.handle), "nvrx_drain")
        slot_a.drained_total = base + total
        engine._staging_free = slot_a.done_event
        lay_a = PackedLayout(shapes=[tuple(t.shape) for t in payload], dtypes=[dtype_name(t.dtype) for t in payload],
                             src_dtypes=[dtype_name(t.dtype) for t in payload], offsets=list(plan.offsets),
                             packed_nbytes=list(plan.packed_nbytes), total_bytes=total)
        snaps.append(Snapshot(engine=engine, slot=slot_a, layout=lay_a, progress_target=slot_a.drained_total, n_total=len(payload)))
        own_views = host_views(lay_a, slot_a.buf)

        xbytes = n * frag_slot
        slot_b = engine._acquire_slot(xbytes)
        base = slot_b.drained_total
        check(engine.lib.nvrx_drain(slot_b.buf.data_ptr, xbuf.ptr, xbytes, engine.drain_chunk, slot_b.buf.progress_ptr, base,
                                    engine._side.handle, slot_b.done_event.handle), "nvrx_drain")
        slot_b.drained_total = base + xbytes
        engine._exchange_free = slot_b.done_event
        frag_views = {m: slot_b.buf.segment(recv_off[m], size, torch.uint8, (size,)) for m, size in zip(self._members, recv_sizes) if m != me}
        lay_b = PackedLayout(shapes=[(s,) for s in recv_sizes if s], dtypes=["uint8"] * sum(1 for s in recv_sizes if s),
                             src_dtypes=["uint8"] * sum(1 for s in recv_sizes if s), offsets=[recv_off[m] for m, s in zip(self._members, recv_sizes) if m != me and s],
                             packed_nbytes=[s for s in recv_sizes if s], total_bytes=xbytes)
        snaps.append(Snapshot(engine=engine, slot=slot_b, layout=lay_b, progress_target=slot_b.drained_total, n_total=len(lay_b.shapes)))
        specs = self._fragment_specs(metas, frag_views, recv_sizes, my_id[0])
        return own_views, specs, snaps

    # ---- load -----------------------------------------------------------------------------------
    @debug_time("ShardedLocalCheckpointManager.load", logger)
    def load(self):
        if self.latest_iteration == -1:
            raise CheckpointingException("The 'find_latest' method must be called before invoking the 'load' function.")
        it = self.latest_iteration
        ckpt_id = self._ckpt_id(it)
        have_own = self._local_ckpt_path_from_id(ckpt_id).exists()
        needs = self.clique.all_gather_object(not have_own)
        result = self._load_fn(ckpt_id) if have_own else None
        for owner, need in zip(self._members, needs):
            if not need:
                continue
            got = self._rebuild_member(it, owner)
            if owner == self.rank:
                result = got
        assert result is not None
        return result, ckpt_id

    def _rebuild_member(self, iteration: int, owner: int):
        """Collective over the clique: every holder sends its fragment of ``owner``; ``owner`` reassembles and scatters."""
        me = self.rank
        n = len(self._members) - 1
        on_gpu = self.clique._payload_on_gpu()
        if me != owner:
            k = self._others(owner).index(me)
            spec = torch.load(self._fragment_path((iteration, owner, k, n)), weights_only=False)
            if k == 0:
                self.clique.send_object({key: spec[key] for key in ("skeleton", "layout", "total_bytes", "shard_bytes")}, owner)
            data = spec["data"]
            if data.numel():
                dist.send(data.cuda() if on_gpu else data, owner, group=self.clique.group)
            return None
        meta = self.clique.recv_object(self._fragment_holder(owner, 0))
        total, sb, layout = meta["total_bytes"], meta["shard_bytes"], meta["layout"]
        skeleton: TensorAwareStateDict = pickle.loads(meta["skeleton"])
        if on_gpu:
            from ...b200 import exchange as xch
            from ...b200.engine import SnapshotEngine

            engine = SnapshotEngine.get()
            staging = engine._ensure_staging(total)
            if engine._staging_free is not None:
                engine._staging_free.synchronize()
            whole = xch.as_uint8_tensor(staging.ptr, total, engine.device)
        else:
            whole = torch.zeros(max(total, 1), dtype=torch.uint8)[:total]
        for k in range(n):
            lo, hi = fragment_range(total, sb, k)
            if hi > lo:
                dist.recv(whole[lo:hi], self._fragment_holder(owner, k), group=self.clique.group)
        skeleton.init_tensors()
        dests = list(skeleton.tensors)
        if on_gpu:
            here = torch.device("cuda", torch.cuda.current_device())
            fixed = [torch.empty_like(d, device=here) if (not d.is_cuda or d.device != here) else d for d in dests]
            if any(f is not d for f, d in zip(fixed, dests)):
                skeleton.pop_tensors()
                skeleton.insert_tensors(fixed)
                dests = fixed
            plan = engine._plan_for(dests, [False] * len(dests))
            assert list(plan.offsets) == list(layout["offsets"]) and plan.staging_bytes == total
            plan.scatter(staging.ptr, engine._current_stream())  # the mirror scatter kernel
            engine.launches += 1 if plan.n_tiles else 0
            torch.cuda.current_stream().synchronize()
        else:
            raw = whole.numpy()
            for d, off, nb in zip(dests, layout["offsets"], layout["nbytes"]):
                if nb:
                    d.copy_(torch.frombuffer(raw[off : off + nb], dtype=d.dtype).view(d.shape))
        return skeleton
