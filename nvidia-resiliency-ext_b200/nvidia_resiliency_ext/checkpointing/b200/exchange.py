"""Packed replica exchange over NCCL / NVLink (the multi-GPU row of the hot path).

Reference (``local/replication/group_utils.py:342-375`` ``all_gather_batch``): for every clique rank, for every
tensor, one ``dist.broadcast`` into a fresh ``torch.empty_like`` followed by ``.to("cpu", non_blocking=True)`` --
F x N NCCL launches and F x N D2H copies.  Here:

    pack kernel  -> this rank's slice of the exchange buffer (HBM)
    ONE all_gather_into_tensor over the clique (NVLink / NVSwitch)
    ONE side-stream drain of the whole exchange buffer -> pinned host slot
    result tensors = views of the slot, per source rank, in that rank's flattening order

``send_packed`` / ``recv_packed`` are the point-to-point analogue used by the retrieve path
(reference ``group_utils.py:378-449``): one packed ``dist.send`` / ``dist.recv`` + one scatter kernel.
"""

from __future__ import annotations

import ctypes as C
import os
import socket
from typing import Optional, Sequence

import torch
import torch.distributed as dist

from ._cabi import check
from .engine import DeviceBuffer, Event, PackedLayout, Snapshot, SnapshotEngine, dtype_name, expected_layout, host_views


class _CudaBytes:
    """``__cuda_array_interface__`` adaptor so c10d can address raw engine memory as a uint8 tensor."""

    def __init__(self, ptr: int, nbytes: int):
        self.__cuda_array_interface__ = {
            "shape": (nbytes,),
            "typestr": "|u1",
            "data": (ptr, False),
            "version": 2,
            "strides": None,
        }


def as_uint8_tensor(ptr: int, nbytes: int, device: int) -> torch.Tensor:
    return torch.as_tensor(_CudaBytes(ptr, max(nbytes, 1)), device=torch.device("cuda", device))[:nbytes]


def _private_buffer(engine: SnapshotEngine, nbytes: int) -> DeviceBuffer:
    """Device scratch for point-to-point payloads (never exported to peers)."""
    buf = getattr(engine, "_p2p_buf", None)
    if buf is None or buf.nbytes < nbytes:
        if buf is not None:
            torch.cuda.current_stream(engine.device).synchronize()
            buf.close()
        buf = DeviceBuffer(max(nbytes, 512), engine.device)
        engine._p2p_buf = buf
    return buf


# ---- the clique-shared exchange buffer and its NVLink peer mappings -----------------------------------
def _drop_peer_maps(engine: SnapshotEngine) -> None:
    maps = getattr(engine, "_peer_maps", None)
    if maps is None:
        engine._peer_maps = {}
        return
    for pm in maps.values():
        for ptr in pm["imported"]:
            engine.lib.nvrx_ipc_close(engine.device, ptr)
    maps.clear()  # in place: callers hold a reference to this dict (re-binding it lost the new entries -> the next
    #               regeneration re-imported handles that were still mapped: cudaErrorAlreadyMapped at 8 ranks)


def _exchange_mode() -> str:
    return os.environ.get("NVRX_B200_EXCHANGE", "auto").lower()  # auto | p2p | nccl


def shared_exchange(engine: SnapshotEngine, group, need: int):
    """Collective over ``group``: the exchange buffer of at least ``need`` bytes on every member and, when the clique
    is NVLink-peer reachable, the device addresses of every member's buffer as seen from this GPU (own included).

    (Re)allocation is decided collectively and ordered: every member first closes the peer mappings it imported, the
    clique synchronises, only then buffers are freed / re-allocated and handles re-exchanged -- an exported allocation is
    never freed while a peer still has it mapped.  Returns ``(buffer, bases or None)``."""
    have = getattr(engine, "_exchange_buf", None)
    have_bytes = have.nbytes if have is not None else 0
    mode = _exchange_mode()
    me = group.my_group_rank
    haves = group.all_gather_int(have_bytes)  # one small tensor collective per exchange; objects only when regenerating
    target = max([need] + haves)
    maps = getattr(engine, "_peer_maps", None)
    if maps is None:
        maps = engine._peer_maps = {}
    key = id(group.group)
    regen = any(h != target for h in haves) or key not in maps
    if regen:
        infos = group.all_gather_object({"host": socket.gethostname(), "boot": _boot_id(), "dev": engine.device})
        free_ev: Optional[Event] = getattr(engine, "_exchange_free", None)
        if free_ev is not None:
            free_ev.synchronize()  # my drain of the buffer (which follows every peer's stores into it) is over
        _drop_peer_maps(engine)
        group.all_gather_int(0)  # everybody closed its imports: exported buffers may now be freed
        if have_bytes != target:
            if have is not None:
                have.close()
            have = engine._exchange_buf = DeviceBuffer(max(target, 512), engine.device)
            engine._exchange_dirty = False  # zero-filled (parity saves rely on it)
        p2p_ok = mode != "nccl" and group.world_size > 1
        p2p_ok = p2p_ok and all(i["host"] == infos[me]["host"] and i["boot"] == infos[me]["boot"] for i in infos)
        # cudaDeviceCanAccessPeer never reports a device as its own peer, but ranks sharing a GPU import each other's
        # buffers through CUDA IPC all the same
        p2p_ok = p2p_ok and all(r == me or i["dev"] == engine.device or torch.cuda.can_device_access_peer(engine.device, i["dev"])
                                for r, i in enumerate(infos))
        votes = group.all_gather_object((bool(p2p_ok), have.ipc_handle() if p2p_ok else None))
        if all(v[0] for v in votes):
            bases, imported = [], []
            for r, (_, handle) in enumerate(votes):
                if r == me:
                    bases.append(have.ptr)
                    continue
                out = C.c_void_p()
                check(engine.lib.nvrx_ipc_import(engine.device, handle, C.byref(out)), "nvrx_ipc_import")
                bases.append(out.value)
                imported.append(out.value)
            maps[key] = {"bases": bases, "imported": imported}
        else:
            if mode == "p2p":
                raise RuntimeError("NVRX_B200_EXCHANGE=p2p but the clique is not NVLink-peer reachable from every member")
            maps[key] = {"bases": None, "imported": []}
    return have, maps[key]["bases"]


def _boot_id() -> str:
    try:
        with open("/proc/sys/kernel/random/boot_id") as f:
            return f.read().strip()
    except OSError:
        return ""


def xor_reduce(engine: SnapshotEngine, dst: int, srcs: Sequence[int], nbytes: int, clear: bool, stream: int) -> None:
    """``dst[0, nbytes) = XOR of the ranges at srcs`` with ONE kernel launch on ``stream`` (``nvrx_xor_reduce``); ``clear``
    zeroes the sources in the same pass."""
    arr = (C.c_void_p * len(srcs))(*srcs)
    check(engine.lib.nvrx_xor_reduce(dst, arr, len(srcs), nbytes, int(clear), stream), "nvrx_xor_reduce")
    engine.launches += 1 if nbytes else 0


def gf_combine(engine: SnapshotEngine, dsts: Sequence[int], srcs: Sequence[int], coef, nbytes: int, clear: bool, stream: int) -> None:
    """``dsts[d][0, nbytes) = sum over s of coef[d][s] * srcs[s]`` in GF(2^8) with ONE kernel launch on ``stream``
    (``nvrx_gf_combine``); ``coef`` is a ``len(dsts) x len(srcs)`` matrix of bytes, ``clear`` zeroes the sources in the
    same pass."""
    flat = bytes(int(c) for row in coef for c in row)
    assert len(flat) == len(dsts) * len(srcs)
    darr = (C.c_void_p * len(dsts))(*dsts)
    sarr = (C.c_void_p * len(srcs))(*srcs)
    carr = (C.c_uint8 * len(flat)).from_buffer_copy(flat)
    check(engine.lib.nvrx_gf_combine(darr, len(dsts), sarr, len(srcs), carr, nbytes, int(clear), stream), "nvrx_gf_combine")
    engine.launches += 1 if nbytes else 0


def _clique_barrier(engine: SnapshotEngine, group) -> None:
    """Stream-ordered barrier over the clique (a 4-byte NCCL all-reduce): no CPU wait."""
    tok = getattr(engine, "_barrier_token", None)
    if tok is None:
        tok = engine._barrier_token = torch.zeros(1, dtype=torch.int32, device=torch.device("cuda", engine.device))
    dist.all_reduce(tok, group=group.group)


def _geometry(group, all_placeholders, align: int, world: int, container: bool = False) -> dict:
    """Per-member layouts inside the exchange buffer, as PackedLayouts and as one union layout; cached on the group for as
    long as the gathered placeholder lists are the same object.  ``container``: every member's slice is laid out in
    checkpoint-container geometry (``ptzip.slot_offsets``), so that it can be drained into a slot of its own and published as
    that member's checkpoint file without a copy."""
    cached = group.__dict__.get("_packed_geometry")
    if (cached is not None and cached["key"] is all_placeholders and cached["align"] == align and cached["world"] == world
            and cached["container"] == container):
        return cached
    layouts = []
    for tps in all_placeholders:
        sizes = [tp.nbytes for tp in tps]
        if container:
            from .ptzip import slot_offsets

            offs, span = slot_offsets(sizes)
            offs, packed, total = list(offs), list(sizes), -(-span // align) * align
        else:
            offs, packed, total = expected_layout(sizes, [False] * len(tps), align)
        layouts.append((offs, packed, total))
    slot_bytes = max(total for _, _, total in layouts)
    slot_bytes = (slot_bytes + 511) // 512 * 512
    dev_lists = []
    for r, (tps, (offs, packed, _)) in enumerate(zip(all_placeholders, layouts)):
        names = [dtype_name(tp.hollow_tensor.dtype) for tp in tps]
        dev_lists.append(
            PackedLayout(
                shapes=[tuple(tp.hollow_tensor.shape) for tp in tps], dtypes=names, src_dtypes=list(names),
                offsets=[r * slot_bytes + o for o in offs], packed_nbytes=list(packed), total_bytes=world * slot_bytes, align=align,
            )
        )
    union = PackedLayout(
        shapes=[s for lay in dev_lists for s in lay.shapes],
        dtypes=[d for lay in dev_lists for d in lay.dtypes],
        src_dtypes=[d for lay in dev_lists for d in lay.src_dtypes],
        offsets=[o for lay in dev_lists for o in lay.offsets],
        packed_nbytes=[n for lay in dev_lists for n in lay.packed_nbytes],
        total_bytes=world * slot_bytes,
        align=align,
    )
    # the same layouts relative to a member's own slice (what a per-member host slot holds)
    own_lists = [
        PackedLayout(shapes=lay.shapes, dtypes=lay.dtypes, src_dtypes=lay.src_dtypes, offsets=list(offs), packed_nbytes=lay.packed_nbytes,
                     total_bytes=total, align=align)
        for lay, (offs, _, total) in zip(dev_lists, layouts)
    ]
    geo = {"key": all_placeholders, "align": align, "world": world, "container": container, "layouts": layouts,
           "slot_bytes": slot_bytes, "dev_lists": dev_lists, "own_lists": own_lists, "union": union}
    group.__dict__["_packed_geometry"] = geo
    return geo


def _container_exchange(engine: SnapshotEngine, group, world: int) -> bool:
    """Zero-copy persistence for replicated saves (opt-in with ``NVRX_B200_ZERO_COPY_REPLICAS=1``, which has to be set on every
    member): possible while the pool of EVERY member can hold one slot per clique member for this save -- the geometry of a
    member's slice is computed by all of them, so the decision is a vote (one small tensor collective, only in this mode)."""
    from .fastsave import replicated_zero_copy_enabled

    if not replicated_zero_copy_enabled():
        return False
    return all(group.all_gather_int(int(engine._spare_slots() >= world)))


def _land_per_member(engine: SnapshotEngine, geo: dict, xbuf, world: int):
    """Drain every member's slice of the exchange buffer into a pinned slot of its own (same bytes over PCIe as one big
    drain), so that each can become that member's checkpoint file by a hard link."""
    from .ptzip import slot_tail_room

    slot_bytes = geo["slot_bytes"]
    result, snaps, last = [], [], None
    for r, lay in enumerate(geo["own_lists"]):
        slot = engine._acquire_slot(slot_bytes + slot_tail_room(len(lay.shapes)))
        base = slot.drained_total
        check(
            engine.lib.nvrx_drain(
                slot.buf.data_ptr, xbuf.ptr + r * slot_bytes, lay.total_bytes, engine.drain_chunk, slot.buf.progress_ptr, base,
                engine._side.handle, slot.done_event.handle,
            ),
            "nvrx_drain",
        )
        slot.drained_total = base + lay.total_bytes
        views = slot.__dict__.get("_exchange_views")
        if views is None or views[0] != slot.buf.name or views[1] is not lay:
            views = slot.__dict__["_exchange_views"] = (slot.buf.name, lay, host_views(lay, slot.buf))
        result.append(list(views[2]))
        snaps.append(Snapshot(engine=engine, slot=slot, layout=lay, progress_target=slot.drained_total, n_total=len(lay.shapes)))
        last = slot
    engine._exchange_free = last.done_event  # the side stream runs the drains in order: the last one ends the reading
    return result, snaps


STREAM_CHUNK = int(os.environ.get("NVRX_B200_STREAM_CHUNK_MB", "256")) << 20


def stream_schedule(slot_bytes: int, chunk_limit: int):
    """``(chunk, [(offset, length, ring half), ...])`` for moving ``slot_bytes`` of every member through the two ring halves:
    chunks are multiples of 512 bytes (the last one may be shorter), alternate between the halves and cover the slice once."""
    chunk = max(512, min(chunk_limit, slot_bytes) // 512 * 512)
    steps = []
    lo = 0
    while lo < slot_bytes:
        ln = min(chunk, slot_bytes - lo)
        steps.append((lo, ln, len(steps) % 2))
        lo += ln
    return chunk, steps


def _allgather_streamed(engine: SnapshotEngine, group, my_tensors, geo: dict, world: int):
    """``NVRX_B200_EXCHANGE=stream`` (opt-in; validated at 2 and 8 GPUs in round 2, tests/test_gpu_multi.py): the exchange leaves the
    training stream.

    The fused / one-shot variants keep an exchange buffer of F x S bytes in HBM (F = clique size, S = snapshot) and run the
    NVLink transfer on the training stream.  Here only the pack does (5 ms for 16 GB, which is what makes the snapshot
    consistent); the packed buffer then travels in chunks, in the background:

        comm stream :  all_gather_into_tensor(ring[c % 2], my staging[chunk c])       NVLink, F x chunk bytes of HBM per half
        drain stream:  ring[c % 2][member r] -> host slot [r * slice + chunk c]        PCIe, starts when chunk c has arrived

    HBM need: S (own staging, as for an unreplicated save) + 2 x F x chunk instead of F x S; the host slot and everything
    behind it (views, writer, files) are the same as for the one-shot exchange."""
    from .engine import Stream, stream_wait_event

    layouts, slot_bytes = geo["layouts"], geo["slot_bytes"]
    me, dev = group.my_group_rank, engine.device
    plan = engine._plan_for(my_tensors, [False] * len(my_tensors))
    assert list(plan.offsets) == layouts[me][0] and plan.staging_bytes == layouts[me][2]
    staging = engine._ensure_staging(slot_bytes)  # padded to the clique-wide slice size: equal-sized all-gathers
    stream = engine._current_stream()
    if engine._staging_free is not None:
        stream_wait_event(stream, engine._staging_free)
    plan.pack(staging.ptr, stream)
    engine.launches += 1 if plan.n_tiles else 0
    packed = Event(dev)
    packed.record(stream)

    chunk, steps = stream_schedule(slot_bytes, STREAM_CHUNK)
    ring = getattr(engine, "_ring_buf", None)
    if ring is None or ring.nbytes < 2 * world * chunk:
        if ring is not None:
            engine._side.synchronize()
            ring.close()
        ring = engine._ring_buf = DeviceBuffer(2 * world * chunk, dev)
    if getattr(engine, "_comm", None) is None:
        engine._comm = Stream(dev)
    comm, drain = engine._comm, engine._side
    comm.wait_event(packed)
    torch_comm = torch.cuda.ExternalStream(comm.handle, device=torch.device("cuda", dev))

    total = world * slot_bytes
    slot = engine._acquire_slot(total)
    base, sent = slot.drained_total, 0
    half_free = [None, None]  # per ring half: recorded after its drains, the next all-gather into it waits for that
    for c, (lo, ln, h) in enumerate(steps):
        half = ring.ptr + h * world * chunk
        if half_free[h] is not None:
            comm.wait_event(half_free[h])
        if world > 1:
            with torch.cuda.stream(torch_comm):
                dist.all_gather_into_tensor(as_uint8_tensor(half, world * ln, dev), as_uint8_tensor(staging.ptr + lo, ln, dev), group=group.group)
            arrived = Event(dev)
            arrived.record(comm.handle)
            drain.wait_event(arrived)
            src0 = half
        else:
            drain.wait_event(packed)
            src0 = staging.ptr + lo
        for r in range(world):
            last = c == len(steps) - 1 and r == world - 1
            check(
                engine.lib.nvrx_drain(
                    slot.buf.data_ptr + r * slot_bytes + lo, src0 + r * ln, ln, engine.drain_chunk, slot.buf.progress_ptr, base + sent,
                    drain.handle, slot.done_event.handle if last else None,
                ),
                "nvrx_drain",
            )
            sent += ln
        freed = Event(dev)
        freed.record(drain.handle)
        half_free[h] = freed
    assert sent == total
    slot.drained_total = base + total
    engine._staging_free = slot.done_event  # the last drain follows the last all-gather, which was the last reader of staging
    engine._exchange_free = slot.done_event
    engine.last_exchange = "nccl-streamed"
    return _views_of_exchange_slot(engine, geo, slot)


def allgather_packed(group, my_tensors: Sequence[torch.Tensor], all_placeholders, target_device):
    """See module docstring.  ``all_placeholders[r]`` describes rank r's tensors (already all-gathered).

    Returns ``(per-rank tensor lists, [Snapshot])``; with a CPU ``target_device`` the tensors are host views that
    become valid once the snapshot has drained."""
    my_tensors = [t.detach() if t.is_contiguous() else t.detach().contiguous() for t in my_tensors]
    engine = SnapshotEngine.get(my_tensors[0].device.index)
    world, me = group.world_size, group.my_group_rank
    align = engine.align

    # everything below that depends only on the clique's tensor structure is computed once per structure: the placeholder
    # lists come from GroupWrapper._gather_placeholders, which hands out the same object while no member's structure changes
    to_host = not (target_device is None or torch.device(target_device).type == "cuda")
    container = to_host and _container_exchange(engine, group, world)
    geo = _geometry(group, all_placeholders, align, world, container)
    layouts, slot_bytes = geo["layouts"], geo["slot_bytes"]
    if to_host and not container and _exchange_mode() == "stream":
        return _allgather_streamed(engine, group, my_tensors, geo, world)

    plan = engine._plan_for(my_tensors, [False] * len(my_tensors), container)
    assert list(plan.offsets) == layouts[me][0] and plan.staging_bytes == layouts[me][2]

    xbuf, bases = shared_exchange(engine, group, world * slot_bytes)
    stream = engine._current_stream()
    free_ev = getattr(engine, "_exchange_free", None)
    if free_ev is not None:
        from .engine import stream_wait_event

        stream_wait_event(stream, free_ev)  # previous drain of the exchange buffer must be over
    whole = as_uint8_tensor(xbuf.ptr, world * slot_bytes, engine.device)
    engine._exchange_dirty = True
    if bases is not None:
        # fused pack + all-gather: ONE kernel reads the tensors once and stores slice `me` into every member's
        # exchange buffer (own HBM + NVLink P2P).  Barrier 1: every member's previous drain of its buffer is over;
        # barrier 2: every member's stores have landed in mine.
        _clique_barrier(engine, group)
        plan.pack_broadcast(bases, me * slot_bytes, stream)
        engine.launches += 1 if plan.n_tiles else 0
        _clique_barrier(engine, group)
        engine.last_exchange = "p2p-fused"
    else:
        plan.pack(xbuf.ptr + me * slot_bytes, stream)
        engine.launches += 1 if plan.n_tiles else 0
        mine = whole[me * slot_bytes : (me + 1) * slot_bytes]
        if world > 1:
            dist.all_gather_into_tensor(whole, mine, group=group.group)
        engine.last_exchange = "nccl-allgather"

    dev_lists = geo["dev_lists"]

    if target_device is None or torch.device(target_device).type == "cuda":
        # stay on the device: hand out copies so the exchange buffer can be reused
        result = [[v.clone() for v in lay.views(whole)] for lay in dev_lists]
        return result, []

    packed_ev = Event(engine.device)
    packed_ev.record(stream)
    engine._side.wait_event(packed_ev)
    if container:
        return _land_per_member(engine, geo, xbuf, world)

    # land everything in ONE pinned host slot with one drain on the side stream
    total = world * slot_bytes
    slot = engine._acquire_slot(total)
    base = slot.drained_total
    check(
        engine.lib.nvrx_drain(
            slot.buf.data_ptr, xbuf.ptr, total, engine.drain_chunk, slot.buf.progress_ptr, base, engine._side.handle,
            slot.done_event.handle,
        ),
        "nvrx_drain",
    )
    slot.drained_total = base + total
    engine._exchange_free = slot.done_event
    return _views_of_exchange_slot(engine, geo, slot)


def _views_of_exchange_slot(engine: SnapshotEngine, geo: dict, slot):
    """Per-member host views of a slot that receives (or received) every member's slice, plus the Snapshot handle."""
    dev_lists = geo["dev_lists"]
    # host views of a (slot buffer, structure) pair are built once: 4 us per tensor is 50 ms for 8 x 1455 tensors otherwise
    views = slot.__dict__.get("_exchange_views")
    if views is None or views[0] != slot.buf.name or views[1] is not dev_lists:
        views = slot.__dict__["_exchange_views"] = (slot.buf.name, dev_lists, [host_views(lay, slot.buf) for lay in dev_lists])
    result = [list(v) for v in views[2]]
    union = geo["union"]
    snap = Snapshot(engine=engine, slot=slot, layout=union, progress_target=slot.drained_total, n_total=len(union.shapes))
    return result, [snap]


def send_packed(group, tensors: Sequence[torch.Tensor], dst_global_rank: int) -> None:
    """Pack ``tensors`` (CUDA, or CPU which are staged through the device first) and send ONE message.  The message
    leaves through ``group.send_tensor``: from the device on NCCL, through host memory on gloo (which sends host memory
    only)."""
    dev = torch.cuda.current_device()
    engine = SnapshotEngine.get(dev)
    cuda_tensors = [t if t.is_cuda else t.to(torch.device("cuda", dev)) for t in tensors]
    cuda_tensors = [t.detach() if t.is_contiguous() else t.detach().contiguous() for t in cuda_tensors]
    plan = engine._plan_for(cuda_tensors, [False] * len(cuda_tensors))
    xbuf = _private_buffer(engine, plan.staging_bytes)
    stream = engine._current_stream()
    plan.pack(xbuf.ptr, stream)
    engine.launches += 1 if plan.n_tiles else 0
    group.send_tensor(as_uint8_tensor(xbuf.ptr, plan.staging_bytes, dev), dst_global_rank)


def recv_packed(group, dests: Sequence[torch.Tensor], src_global_rank: int) -> None:
    """Receive ONE packed message and scatter it into ``dests`` (CUDA tensors, or CPU tensors filled through a
    device bounce as the reference does at ``group_utils.py:442-446``).  The message arrives through
    ``group.recv_tensor``: straight into device memory on NCCL, through a host buffer on gloo."""
    dev = torch.cuda.current_device()
    engine = SnapshotEngine.get(dev)
    on_dev = [d if d.is_cuda else torch.empty(d.shape, dtype=d.dtype, device=torch.device("cuda", dev)) for d in dests]
    assert all(d.is_contiguous() for d in on_dev)
    plan = engine._plan_for(on_dev, [False] * len(on_dev))
    xbuf = _private_buffer(engine, plan.staging_bytes)
    group.recv_tensor(as_uint8_tensor(xbuf.ptr, plan.staging_bytes, dev), src_global_rank)
    stream = engine._current_stream()
    plan.scatter(xbuf.ptr, stream)
    engine.launches += 1 if plan.n_tiles else 0
    for d, o in zip(dests, on_dev):
        if not d.is_cuda:
            d.copy_(o)
    torch.cuda.current_stream(dev).synchronize()
