"""``torch.save`` whose tensor payload is written by a pool of ``pwrite`` workers straight from snapshot slots.

Stock ``torch.save`` pushes every storage through one thread (memcpy into the zip stream + crc32).  Here the
container is produced by PyTorch itself with its data records *skipped* (``torch.serialization.skip_data``, a
sparse file that already has every header, ``data.pkl`` and the central directory), and the records are then
filled in place from the pinned shared-memory slot by ``nvrx_hostbuf_writev_fd``.  The result is an ordinary
checkpoint file: ``torch.load`` (plain or ``mmap=True``) reads it, and it is record-for-record what
``torch.save`` of the same object would have laid out.

Replaces the payload part of the reference's single-threaded writer
(``local/ckpt_managers/local_manager.py:117-122``, ``async_ckpt/torch_ckpt.py:36-41``).  CPU only; never calls CUDA.
"""

from __future__ import annotations

import ctypes as C
import os
import pickle
from contextlib import contextmanager
from typing import List, Sequence, Tuple

import torch

from .persist import zip_crc_enabled

WRITE_THREADS = int(os.environ.get("NVRX_B200_WRITE_THREADS", "16"))

# (base address, capacity, HostBuffer) ranges the current writer may find tensor storages in
_active_ranges: List[Tuple[int, int, object]] = []


@contextmanager
def slot_ranges(ranges: Sequence[Tuple[int, int, object]]):
    """Declare the snapshot slots tensors may live in while saving (used by the managers' writer functions)."""
    ranges = list(ranges)
    _active_ranges.extend(ranges)
    try:
        yield
    finally:
        if ranges:
            del _active_ranges[-len(ranges) :]


def ranges_for(descs, held) -> List[Tuple[int, int, object]]:
    """Address ranges for the snapshot descriptors ``descs`` whose slots are mapped as ``held`` in this process.
    A forked writer also sees the trainer's mapping (tensor views were created there) at the trainer's address."""
    out = []
    for desc, hb in zip(descs, held):
        hb.crc_info = desc.get("crc")  # where the GPU left checksum values for this snapshot, if it did
        out.append((hb.data_ptr, hb.capacity, hb))
        base = desc.get("owner_base")
        if base and base != hb.data_ptr and desc.get("owner_pid") in (os.getppid(), os.getpid()):
            out.append((base, hb.capacity, hb))
    return out


class _RecordingZip:
    """Stands in for PyTorchFileWriter during a dry run of the pickler: remembers which storage became which
    ``data/<key>`` record (by address), copies nothing."""

    def __init__(self):
        self.records: List[Tuple[str, int, int]] = []

    def write_record(self, name, data, nbytes):
        if name.startswith("data/") and not isinstance(data, (str, bytes)):
            self.records.append((name, data.data_ptr(), int(nbytes)))

    def write_record_metadata(self, name, nbytes):  # pragma: no cover - not used in the dry run
        self.records.append((name, 0, int(nbytes)))


def _locate(ptr: int, nbytes: int):
    for base, cap, hb in _active_ranges:
        if base <= ptr and ptr + nbytes <= base + cap:
            return hb, ptr - base
    return None, 0


def zero_copy_enabled() -> bool:
    """Default ON (tests/test_gpu_zzero_copy.py): snapshots are packed in checkpoint-container
    geometry and a save whose target shares a file system with the slots (``/dev/shm``) publishes the slot with a hard link
    instead of copying it -- writing 16 GB into a fresh tmpfs file is bounded by the kernel's page allocation whatever
    the number of writers, the link takes milliseconds.  Targets on other file systems, state dicts
    with host tensors and saves that would take the last unpublished slot fall back to the copying writer by themselves.
    ``NVRX_B200_ZERO_COPY=0`` always copies (a published file shares its pages with the slot, see DESIGN.md for the caveat)."""
    return os.environ.get("NVRX_B200_ZERO_COPY", "1") != "0"


def replicated_zero_copy_enabled() -> bool:
    """Opt-in (``NVRX_B200_ZERO_COPY_REPLICAS=1``, on every clique member): the replica exchange drains every member's slice
    into a slot of its own so that replicas are published by hard links as well (b200/exchange.py)."""
    return zero_copy_enabled() and os.environ.get("NVRX_B200_ZERO_COPY_REPLICAS", "0") == "1"


def _gpu_crcs(slot, info: dict, offsets, sizes) -> List[int]:
    """Record checksums from the partial values a kernel left behind the payload (``nvrx_crc_run``): wait for the ready word
    (CPU only, like the drain's progress word), then chain values and left-over bytes (``nvrx_crc_finish``)."""
    import time

    from .engine import finish_crcs
    from .persist import DRAIN_TIMEOUT_MS

    ready = C.c_uint64.from_address(slot.data_ptr + info["ready_offset"])
    deadline = time.monotonic() + DRAIN_TIMEOUT_MS / 1e3
    while ready.value != info["ready_value"]:
        if time.monotonic() > deadline:
            raise TimeoutError("checksum values of the snapshot did not arrive")
        time.sleep(0.0002)
    return finish_crcs(offsets, sizes, slot.data_ptr + info["offset"], info["n_values"], slot.data_ptr)


def _locate_or_none(ptr: int, nbytes: int):
    hb, off = _locate(ptr, nbytes)
    return None if hb is None else (hb, off)


def _single_slot(records):
    """``(slot, offsets, sizes)`` when the storages of the object are ``data/0..n-1`` and every non-empty one lives in ONE named
    snapshot slot; else ``(None, [], [])``."""
    if [r[0] for r in records] != [f"data/{i}" for i in range(len(records))]:
        return None, [], []
    slot, offsets, sizes = None, [], []
    for _, ptr, nbytes in records:
        hb, off = _locate(ptr, nbytes) if nbytes else (slot, 0)
        if nbytes:
            if hb is None or not hb.name or (slot is not None and hb.name != slot.name):
                return None, [], []
            slot = hb
        offsets.append(off)
        sizes.append(nbytes)
    return slot, offsets, sizes


def _try_link(obj, target: str, records, protocol) -> bool:
    """Publish the snapshot slot itself as the checkpoint file (``ptzip.publish_slot``) when every tensor of ``obj`` lives
    in ONE named slot, in storage order, at the container's offsets.  False = nothing published, copy instead."""
    from . import ptzip

    slot, offsets, sizes = _single_slot(records)
    if slot is None or not hasattr(torch.serialization, "skip_data"):
        return False
    crcs = None
    info = getattr(slot, "crc_info", None)
    if info:
        crcs = _gpu_crcs(slot, info, offsets, sizes)
    elif zip_crc_enabled():
        crcs = slot.crc32v(offsets, sizes, WRITE_THREADS)
    small = ptzip.small_records(obj, protocol)
    keep = info["ready_offset"] + 8 if info else 0  # the values stay readable in the published file's pad area
    return ptzip.publish_slot("/dev/shm" + slot.name, target, small, offsets, sizes, crcs=crcs, keep_until=keep)


def save(obj, f, *args, **kwargs) -> str:
    """Drop-in for ``torch.save(obj, f, ...)``.  Returns which path was taken: "linked" (zero-copy publish of the slot),
    "parallel" (container by PyTorch, payload by the slot's writer pool) or "torch"."""
    if not _active_ranges or args or set(kwargs) - {"pickle_protocol"} or not hasattr(torch.serialization, "skip_data"):
        torch.save(obj, f, *args, **kwargs)
        return "torch"
    protocol = kwargs.get("pickle_protocol", torch.serialization.DEFAULT_PROTOCOL)
    try:
        dry = _RecordingZip()
        torch.serialization._save(obj, dry, pickle, protocol, False)
        records = dry.records
    except Exception:  # noqa: BLE001 - private API moved: use the stock writer
        torch.save(obj, f, **kwargs)
        return "torch"

    is_path = isinstance(f, (str, os.PathLike))
    start = 0 if is_path else f.tell()
    if zero_copy_enabled() and start == 0:
        target = os.fspath(f) if is_path else getattr(f, "name", None)
        # a file object was opened (exclusively, by the managers) on its name: the link replaces that empty file
        if isinstance(target, str) and _try_link(obj, target, records, protocol):
            return "linked"
    named = os.fspath(f) if is_path else getattr(f, "name", None)
    if start == 0 and isinstance(named, str):
        # the GPU summed the records while the snapshot drained (opt-in): write our own payload-first container, whose headers
        # take those checksums -- PyTorch's writer would either leave them zero or sum 16 GB on one core.  (A file object was
        # opened on its name by the caller, exclusively in the managers' case; the container is written through the name.)
        slot, offsets, sizes = _single_slot(records)
        info = getattr(slot, "crc_info", None) if slot is not None else None
        if info and protocol == torch.serialization.DEFAULT_PROTOCOL and hasattr(torch.serialization, "skip_data"):
            from . import ptzip

            ptzip.save(obj, named, locate=_locate_or_none, threads=WRITE_THREADS, crcs=_gpu_crcs(slot, info, offsets, sizes))
            return "parallel+gpu-crc"
    name = named
    if start != 0 or not isinstance(name, str) or (not is_path and not os.path.exists(name)):
        # an unnamed file object (BytesIO, pipe) or a write that does not start the file: nothing the parallel writer can fill
        # in by offset -- the stock writer handles those (checked BEFORE anything is emitted into f)
        torch.save(obj, f, **kwargs)
        return "torch"
    # A path is filled under a private name and renamed into place when complete: several ranks saving to ONE path (the
    # reference's own test does, tests/checkpointing/unit/test_async_save.py:38) must not truncate the file another writer
    # has mapped (SIGBUS in that writer), and readers never see a half-written checkpoint.
    final = scratch = None
    if is_path:
        # (same base name inside a scratch directory: PyTorch names the archive inside the zip after the file)
        scratch = os.path.join(os.path.dirname(os.path.abspath(name)), f".nvrx_tmp_{os.getpid()}_{os.urandom(4).hex()}")
        os.mkdir(scratch)
        final, name = name, os.path.join(scratch, os.path.basename(name))
        f = name
    try:
        with torch.serialization.skip_data():
            torch.save(obj, f, **kwargs)
    except BaseException:
        if scratch is not None:
            import shutil

            shutil.rmtree(scratch, ignore_errors=True)
        raise
    if not is_path:
        f.flush()
    reader = torch._C.PyTorchFileReader(os.fspath(name))
    fd = os.open(name, os.O_RDWR)  # a descriptor of our own, read+write: the writer maps the range, the checksum patch reads
    ok = False
    try:
        by_slot = {}
        patch, patch_crcs = [], []  # records whose checksum is known here: (name, data offset, size)
        want_crc = zip_crc_enabled()
        for rec, ptr, nbytes in records:
            if nbytes == 0:
                continue
            file_off = reader.get_record_offset(rec)
            hb, off = _locate(ptr, nbytes)
            if hb is None:  # a tensor that does not live in a snapshot slot (pass-through host tensor)
                raw = C.string_at(ptr, nbytes)
                os.pwrite(fd, raw, file_off)
                if want_crc:
                    import zlib

                    patch.append((rec, file_off, nbytes))
                    patch_crcs.append(zlib.crc32(raw))
                continue
            ent = by_slot.setdefault(id(hb), (hb, [], [], [], []))
            ent[1].append(off)
            ent[2].append(nbytes)
            ent[3].append(file_off)
            ent[4].append(rec)
        for hb, offs, sizes, file_offs, names in by_slot.values():
            hb.writev_fd(offs, sizes, file_offs, fd, WRITE_THREADS)
            if want_crc:
                # skip_data left the data records' checksums zero: sum the slot (not the file) with the writer pool and patch
                patch.extend(zip(names, file_offs, sizes))
                patch_crcs.extend(hb.crc32v(offs, sizes, WRITE_THREADS))
        if patch:
            from . import ptzip

            ptzip.patch_record_crcs(fd, patch, patch_crcs)
        ok = True
    finally:
        del reader
        os.close(fd)
        if final is not None:
            try:
                if ok:
                    os.replace(name, final)
                else:
                    os.unlink(name)
            finally:
                try:
                    os.rmdir(scratch)
                except OSError:
                    pass
    return "parallel"
