"""A ``torch.load``-able checkpoint container whose tensor payload sits at offsets WE choose.

PyTorch checkpoints are ZIP archives of *stored* (uncompressed) records; ``torch.load`` finds records through the central
directory, so the order of records in the file is free.  ``torch.save`` puts ``data.pkl`` first, which makes every payload
offset depend on the size of the pickle.  This writer inverts that:

    [ local header | data/0 ] [ local header | data/1 ] ...      <- payload region: offsets depend only on tensor sizes
    [ data.pkl ] [ byteorder ] [ version ] ...                   <- small records, whatever PyTorch would have written
    [ pad record ] [ central directory ] [ zip64 EOCD ] [ EOCD ] <- the tail can be pinned to the end of a fixed-size file

so the payload region of the *file* can have the same geometry as the packed staging buffer of the snapshot engine.  It is
the host half of zero-copy persistence (DESIGN.md "next"): the pinned host slot a snapshot drains into can be the tmpfs
checkpoint file itself.  This module is CPU-only and self-contained; today it is exercised by ``tests/test_ptzip_cpu.py``
and not yet on the default save path (that needs the file-backed slot to be validated on a GPU box).

Small records (pickle with PyTorch's persistent-id scheme, ``version``, ``byteorder``, ...) are produced by PyTorch itself:
``torch.save`` with ``skip_data`` into memory, read back record by record -- nothing about their content is hard-coded here.
"""

from __future__ import annotations

import io
import os
import pickle
import struct
import zlib
from dataclasses import dataclass, field
from typing import Any, Callable, List, Optional, Sequence, Tuple

import torch

ALIGN = 64  # PyTorch aligns record data to 64 bytes (mmap-friendly)
_PAD_ID = 0x4246  # "FB": the extra-field id PyTorch uses for its alignment padding
_U32 = 0xFFFFFFFF


@dataclass
class Record:
    name: str  # full name inside the archive ("<archive>/data/0")
    size: int
    header_off: int = 0
    data_off: int = 0
    crc: int = 0


@dataclass
class PayloadLayout:
    """Where every storage record lives; a function of (archive name, storage sizes) only."""

    archive: str
    records: List[Record] = field(default_factory=list)
    end: int = 0  # first byte after the last payload record


def _local_header(name: bytes, size: int, crc: int, data_off_hint: int, header_off: int, force_zip64: bool) -> bytes:
    """Local file header whose extra field pads the record data to ``ALIGN`` (and carries zip64 sizes when needed)."""
    zip64 = force_zip64 or size >= _U32
    extra = b""
    if zip64:
        extra += struct.pack("<HHQQ", 0x0001, 16, size, size)
    fixed = 30 + len(name)
    pad_to = data_off_hint - header_off - fixed - len(extra)
    assert pad_to >= 4 or pad_to == 0, pad_to
    if pad_to:
        extra += struct.pack("<HH", _PAD_ID, pad_to - 4) + b"Z" * (pad_to - 4)
    hdr = struct.pack(
        "<IHHHHHIIIHH", 0x04034B50, 45 if zip64 else 20, 0, 0, 0, 0x21, crc & _U32,
        _U32 if zip64 else size, _U32 if zip64 else size, len(name), len(extra),
    )
    return hdr + name + extra


def _data_offset_after(header_off: int, name_len: int, zip64: bool, align: int = ALIGN) -> int:
    """Smallest ``align``-aligned data offset that leaves room for the header (+ zip64 extra) and a legal padding field."""
    need = header_off + 30 + name_len + (20 if zip64 else 0)
    off = -(-need // align) * align
    while 0 < off - need < 4:  # a padding extra field needs at least its 4-byte header
        off += align
    return off


def plan_payload(archive: str, sizes: Sequence[int], *, start: int = 0, force_zip64: bool = False, align: int = ALIGN) -> PayloadLayout:
    """Lay out ``data/<i>`` records of the given sizes starting at file offset ``start``; record data is aligned to
    ``align`` (a multiple of PyTorch's 64)."""
    assert align % ALIGN == 0
    lay = PayloadLayout(archive=archive)
    cur = start
    for i, size in enumerate(sizes):
        name = f"{archive}/data/{i}"
        zip64 = force_zip64 or size >= _U32
        data_off = _data_offset_after(cur, len(name.encode()), zip64, align)
        lay.records.append(Record(name=name, size=size, header_off=cur, data_off=data_off))
        cur = data_off + size
    lay.end = cur
    return lay


class _Recorder:
    """Dry-run stand-in for PyTorchFileWriter: which storage became which ``data/<key>`` record."""

    def __init__(self):
        self.storages: List[Tuple[str, int, int]] = []

    def write_record(self, name, data, nbytes):
        if name.startswith("data/") and not isinstance(data, (str, bytes)):
            self.storages.append((name, data.data_ptr(), int(nbytes)))

    def write_record_metadata(self, name, nbytes):  # pragma: no cover
        self.storages.append((name, 0, int(nbytes)))


def describe(obj: Any, protocol: int = torch.serialization.DEFAULT_PROTOCOL) -> Tuple[List[Tuple[str, bytes]], List[Tuple[int, int]]]:
    """``(small_records, storages)`` of ``obj`` as PyTorch would serialise it.

    small_records: ``[(record name without archive prefix, bytes)]`` for everything that is not tensor data, in PyTorch's
    order; storages: ``[(data_ptr, nbytes)]`` in key order (``data/0``, ``data/1``, ...)."""
    rec = _Recorder()
    torch.serialization._save(obj, rec, pickle, protocol, False)
    keys = [int(n.split("/", 1)[1]) for n, _, _ in rec.storages]
    assert keys == list(range(len(keys))), "storage keys are expected to be 0..n-1 in order"
    return small_records(obj, protocol), [(ptr, nb) for _, ptr, nb in rec.storages]


def _central_entry(name: bytes, size: int, crc: int, header_off: int, force_zip64: bool) -> bytes:
    z_size = force_zip64 or size >= _U32
    z_off = force_zip64 or header_off >= _U32
    extra = b""
    if z_size or z_off:
        body = b""
        if z_size:
            body += struct.pack("<QQ", size, size)
        if z_off:
            body += struct.pack("<Q", header_off)
        extra = struct.pack("<HH", 0x0001, len(body)) + body
    need = 45 if (z_size or z_off) else 20
    return struct.pack(
        "<IHHHHHHIIIHHHHHII", 0x02014B50, need, need, 0, 0, 0, 0x21, crc & _U32,
        _U32 if z_size else size, _U32 if z_size else size, len(name), len(extra), 0, 0, 0, 0,
        _U32 if z_off else header_off,
    ) + name + extra


_PAD_CRC_LIMIT = 256 << 20


def _crc_of_file_range(fd: int, off: int, n: int) -> int:
    crc, step = 0, 8 << 20
    while n > 0:
        chunk = os.pread(fd, min(step, n), off)
        if not chunk:  # beyond EOF of a sparse file: zeros
            chunk = bytes(min(step, n))
        crc = zlib.crc32(chunk, crc)
        off += len(chunk)
        n -= len(chunk)
    return crc & _U32


def small_records(obj: Any, protocol: int = torch.serialization.DEFAULT_PROTOCOL) -> List[Tuple[str, bytes]]:
    """Everything PyTorch writes for ``obj`` besides tensor data (``data.pkl``, ``byteorder``, ``version``, ...).

    PyTorch itself produces them: ``torch.save`` with the data skipped into a scratch FILE, which the writer leaves sparse
    (it seeks over the records).  An in-memory ``BytesIO`` target must not be used here: seeking over 16 GB of skipped records
    and then writing makes it allocate and zero all of it (seconds per checkpoint)."""
    import tempfile

    scratch_dir = "/dev/shm" if os.access("/dev/shm", os.W_OK) else None
    with tempfile.NamedTemporaryFile(dir=scratch_dir, prefix="nvrx_b200_skel_", suffix=".pt") as tf:
        with torch.serialization.skip_data():
            torch.save(obj, tf.name, pickle_protocol=protocol)
        reader = torch._C.PyTorchFileReader(tf.name)
        out = [(n, bytes(reader.get_record(n))) for n in reader.get_all_records() if not n.startswith("data/")]
        del reader
    return out


def tail_size(archive: str, small: Sequence[Tuple[str, bytes]], n_storages: int, force_zip64: bool = False) -> int:
    """Upper bound of the bytes needed after the payload region (small records + pad record + directory + EOCDs)."""
    names = [f"{archive}/{n}" for n, _ in small] + [f"{archive}/data/{i}" for i in range(n_storages)] + [f"{archive}/.pad"]
    local = sum(30 + len(n.encode()) + 20 + ALIGN + 4 for n in names[: len(small)] + names[-1:]) + sum(len(b) for _, b in small)
    central = sum(46 + len(n.encode()) + 28 for n in names)
    return local + central + 56 + 20 + 22 + 2 * ALIGN


def write_container(
    fd: int,
    layout: PayloadLayout,
    small: Sequence[Tuple[str, bytes]],
    *,
    file_size: Optional[int] = None,
    crcs: Optional[Sequence[int]] = None,
    write_payload: Optional[Callable[[Record], None]] = None,
    force_zip64: bool = False,
    pad_crc: bool = True,
) -> int:
    """Write headers, small records, pad record, central directory and EOCDs around a payload region planned by
    :func:`plan_payload`.  Payload bytes themselves are NOT written unless ``write_payload(record)`` is given (they may
    already be there: the region can be the destination of a DMA).

    ``file_size``: when set, the archive is made to end exactly there (a ``.pad`` record absorbs the slack), so a fixed-size
    pre-pinned file can be reused for snapshots of any smaller size.  Returns the archive end offset.
    ``crcs[i]``: crc32 of storage i (0 when omitted -- ``torch.load`` does not verify; ``zipfile.testzip`` would)."""
    archive = layout.archive
    central: List[bytes] = []
    # payload records: headers only
    for i, rec in enumerate(layout.records):
        rec.crc = (crcs[i] if crcs is not None else 0) & _U32
        name = rec.name.encode()
        os.pwrite(fd, _local_header(name, rec.size, rec.crc, rec.data_off, rec.header_off, force_zip64), rec.header_off)
        if write_payload is not None and rec.size:
            write_payload(rec)
        central.append(_central_entry(name, rec.size, rec.crc, rec.header_off, force_zip64))
    cur = layout.end
    # small records (PyTorch's own bytes)
    for n, data in small:
        name = f"{archive}/{n}".encode()
        crc = zlib.crc32(data) & _U32
        data_off = _data_offset_after(cur, len(name), force_zip64)
        os.pwrite(fd, _local_header(name, len(data), crc, data_off, cur, force_zip64), cur)
        os.pwrite(fd, data, data_off)
        central.append(_central_entry(name, len(data), crc, cur, force_zip64))
        cur = data_off + len(data)
    n_entries = len(central)
    cd_bytes = b"".join(central)
    tail_fixed = 56 + 20 + 22
    if file_size is not None:
        # a ".pad" record soaks up the slack so that the EOCD is the last thing in the file
        name = f"{archive}/.pad".encode()
        pad_central_len = 46 + len(name) + 28
        data_off = _data_offset_after(cur, len(name), True)
        slack = file_size - data_off - (len(cd_bytes) + pad_central_len + tail_fixed)
        if slack < 0:
            raise ValueError(f"file_size {file_size} too small for the container (short by {-slack} bytes)")
        pad_entry = _central_entry(name, slack, 0, cur, True)
        # the central entry was budgeted with the largest zip64 extra; make up the difference with a longer pad
        slack += pad_central_len - len(pad_entry)
        # the pad covers whatever the file holds there (zeros in a fresh file, stale bytes in a reused slot); its crc is
        # only computed when that is cheap -- nothing ever reads the record, it exists to keep the EOCD at the file end
        pad_sum = _crc_of_file_range(fd, data_off, slack) if pad_crc and slack <= _PAD_CRC_LIMIT else 0
        pad_entry = _central_entry(name, slack, pad_sum, cur, True)
        os.pwrite(fd, _local_header(name, slack, pad_sum, data_off, cur, True), cur)
        cd_bytes += pad_entry
        n_entries += 1
        cur = data_off + slack
    cd_off = cur
    os.pwrite(fd, cd_bytes, cd_off)
    cur = cd_off + len(cd_bytes)
    # zip64 end of central directory + locator (always written: payloads are routinely > 4 GiB), then the classic EOCD
    z64 = struct.pack("<IQHHIIQQQQ", 0x06064B50, 44, 45, 45, 0, 0, n_entries, n_entries, len(cd_bytes), cd_off)
    loc = struct.pack("<IIQI", 0x07064B50, 0, cur, 1)
    eocd = struct.pack(
        "<IHHHHIIH", 0x06054B50, 0, 0, min(n_entries, 0xFFFF), min(n_entries, 0xFFFF),
        min(len(cd_bytes), _U32), min(cd_off, _U32), 0,
    )
    os.pwrite(fd, z64 + loc + eocd, cur)
    end = cur + len(z64) + len(loc) + len(eocd)
    if file_size is not None:
        assert end == file_size, (end, file_size)
    return end


def save(obj: Any, path, *, locate: Callable[[int, int], Optional[Tuple[Any, int]]], threads: int = 16,
         compute_crc: bool = True, file_size: Optional[int] = None, force_zip64: bool = False,
         crcs: Optional[Sequence[int]] = None) -> PayloadLayout:
    """Write ``obj`` as a checkpoint with the payload-first layout.  ``locate(data_ptr, nbytes)`` maps a storage to
    ``(HostBuffer, offset)`` (payload copied by the buffer's parallel writer) or ``None`` (copied from process memory).
    ``crcs``: record checksums that are already known (one per storage, e.g. from the GPU) -- nothing is summed here then."""
    import ctypes as C

    small, storages = describe(obj)
    archive = os.path.splitext(os.path.basename(os.fspath(path)))[0] or "archive"
    layout = plan_payload(archive, [nb for _, nb in storages], force_zip64=force_zip64)
    fd = os.open(path, os.O_CREAT | os.O_RDWR | os.O_TRUNC, 0o644)
    try:
        total = file_size if file_size is not None else layout.end + tail_size(archive, small, len(storages), force_zip64)
        os.ftruncate(fd, total)
        known = list(crcs) if crcs is not None else None
        assert known is None or len(known) == len(storages)
        compute_crc = compute_crc and known is None
        crcs, by_buf = [], {}
        for rec, (ptr, nb) in zip(layout.records, storages):
            hit = locate(ptr, nb) if nb else None
            if hit is None:
                raw = C.string_at(ptr, nb) if nb else b""
                os.pwrite(fd, raw, rec.data_off)
                crcs.append(zlib.crc32(raw) if compute_crc else 0)
            else:
                hb, off = hit
                ent = by_buf.setdefault(id(hb), (hb, [], [], []))
                ent[1].append(off)
                ent[2].append(nb)
                ent[3].append(rec.data_off)
                crcs.append(hb.crc32(off, nb, threads) if compute_crc else 0)
        for hb, offs, sizes, file_offs in by_buf.values():
            hb.writev_fd(offs, sizes, file_offs, fd, threads)
        end = write_container(fd, layout, small, file_size=file_size, crcs=known if known is not None else crcs, force_zip64=force_zip64)
        if file_size is None:
            os.ftruncate(fd, end)
    finally:
        os.close(fd)
    return layout


# --------------------------------------------------------------------------------------------------
# slot geometry: a snapshot slot that is a checkpoint file
# --------------------------------------------------------------------------------------------------
# A host snapshot slot is a POSIX shm object = a file on the /dev/shm tmpfs: [ 4096-byte header page | payload ].  The
# header page starts with a ZIP local file header (csrc/hostbuf.cu::write_slot_prefix), so when the payload region was
# packed at the offsets ``slot_offsets`` gives, the slot becomes a valid checkpoint by writing headers into the gaps and the
# tail at the end of the file -- and is *published* with a hard link instead of a copy.
SLOT_PREFIX = 4096
SLOT_ARCHIVE = "archive"  # what torch.save calls the archive when it is given a buffer
SLOT_ALIGN = 512  # == the engine's default segment alignment, so the kernels see the geometry they were tuned on


def slot_layout(sizes: Sequence[int]) -> PayloadLayout:
    return plan_payload(SLOT_ARCHIVE, sizes, start=SLOT_PREFIX, align=SLOT_ALIGN)


def slot_offsets(sizes: Sequence[int]) -> Tuple[List[int], int]:
    """Payload-relative offsets for segments of the given (packed) sizes, and the payload bytes they span."""
    lay = slot_layout(sizes)
    return [r.data_off - SLOT_PREFIX for r in lay.records], lay.end - SLOT_PREFIX


def slot_tail_room(n_storages: int) -> int:
    """Bytes to keep free after the payload for small records + directory.  A guess (the pickle is not known when the slot
    is sized); a tail that does not fit makes ``publish_slot`` decline and the caller copies instead."""
    return (1 << 20) + 1024 * n_storages


def publish_slot(
    slot_path: str,
    target: str,
    small: Sequence[Tuple[str, bytes]],
    offsets: Sequence[int],
    sizes: Sequence[int],
    *,
    crcs: Optional[Sequence[int]] = None,
    keep_until: int = 0,
) -> bool:
    """Turn the slot file ``slot_path`` into the checkpoint ``target`` without copying its payload.

    ``keep_until``: payload-relative end of a region behind the storages that must stay intact (the GPU's checksum values);
    the small records start after it.

    ``offsets[i]`` / ``sizes[i]``: where storage ``i`` sits in the payload region.  Returns False (nothing changed that
    matters: only bytes outside the storages are written) when the geometry is not the container's, the tail does not
    fit, or the two paths cannot be hard-linked (different file systems).  An existing ``target`` is replaced atomically."""
    lay = slot_layout(sizes)
    for rec, off, size in zip(lay.records, offsets, sizes):
        if size and off != rec.data_off - SLOT_PREFIX:
            return False
    lay.end = max(lay.end, SLOT_PREFIX + keep_until)
    try:
        fd = os.open(slot_path, os.O_RDWR)
    except OSError:
        return False
    try:
        file_size = os.fstat(fd).st_size
        if lay.end + tail_size(SLOT_ARCHIVE, small, len(sizes)) > file_size:
            return False
        # with checksummed storages the pad is checksummed too (up to _PAD_CRC_LIMIT, as in a copied file): a record with
        # a zero checksum makes zipfile.testzip() / unzip -t report the whole checkpoint as corrupt
        write_container(fd, lay, small, file_size=file_size, crcs=crcs, pad_crc=crcs is not None)
    finally:
        os.close(fd)
    # temporary link name: keeps the target's extension so that a manager's cleanup glob (iter_*_local*.pt) also removes a
    # leftover from a writer that died between the two calls below (it would pin the slot forever otherwise)
    root, ext = os.path.splitext(os.fspath(target))
    tmp = f"{root}.nvrx{os.getpid()}{ext}"
    try:
        if os.path.lexists(tmp):
            os.unlink(tmp)
        os.link(slot_path, tmp)
        os.replace(tmp, target)
    except OSError:
        return False
    return True


def slot_is_published(slot_path: str) -> bool:
    """True while some checkpoint file is a hard link to this slot (its pages must not be overwritten)."""
    try:
        return os.stat(slot_path).st_nlink > 1
    except OSError:
        return False


def _mapping_base(path, ptr: int) -> Optional[int]:
    """Address at which offset 0 of ``path`` is mapped in this process, taken from the mapping that contains ``ptr``
    (``/proc/self/maps``); None when no mapping of that file contains it."""
    try:
        real = os.path.realpath(os.fspath(path))
        st = os.stat(real)
        with open("/proc/self/maps") as f:
            for line in f:
                parts = line.split(None, 5)
                if len(parts) < 6:
                    continue
                lo, hi = (int(x, 16) for x in parts[0].split("-"))
                if not lo <= ptr < hi:
                    continue
                name = parts[5].rstrip("\n")
                if name.endswith(" (deleted)"):
                    name = name[: -len(" (deleted)")]
                try:
                    same = name == real or os.path.samestat(os.stat(name), st)
                except OSError:
                    same = False
                return lo - int(parts[2], 16) if same else None
    except (OSError, ValueError):
        pass
    return None


def tensor_offsets_in_file(path, tensors: Sequence[torch.Tensor]) -> Optional[List[int]]:
    """File offsets of the data of ``tensors`` -- tensors ``torch.load(path, mmap=True)`` returned, in ascending file order --
    or None when they are not views of the data records of one mapping of that file, ascending and 16-byte aligned.

    The address the file is mapped at comes from ``/proc/self/maps`` (exact).  Every tensor must then start at the data offset
    of a ``data/<k>`` record that is large enough: usually record i for tensor i, but objects that pickle other storages first
    (a host tensor in the ``common`` part of a Megatron-style state dict) shift the numbering.  Without a usable maps entry the
    base is inferred from the records (tensor i = record i, else the one base under which every tensor hits a record)."""
    live = [(i, t) for i, t in enumerate(tensors) if t.numel()]
    if not live or any(t.is_cuda or not t.is_contiguous() for _, t in live):
        return None
    try:
        reader = torch._C.PyTorchFileReader(os.fspath(path))
        recs = {}
        for name in reader.get_all_records():
            if name.startswith("data/"):
                recs[reader.get_record_offset(name)] = name
        first_i, first_t = live[0]

        def fits(guess: int) -> bool:
            return all((t.data_ptr() - guess) in recs for _, t in live)

        base = _mapping_base(path, first_t.data_ptr())
        if base is not None and not fits(base):
            return None
        if base is None and reader.has_record(f"data/{first_i}"):
            guess = first_t.data_ptr() - reader.get_record_offset(f"data/{first_i}")
            if len(live) > 1 and all(reader.has_record(f"data/{i}") and reader.get_record_offset(f"data/{i}") == t.data_ptr() - guess for i, t in live):
                base = guess
        if base is None:
            if len(live) < 2:
                return None  # one tensor fits under every record: only the maps entry can place it
            candidates = [first_t.data_ptr() - off0 for off0 in sorted(recs)]
            good = [g for g in candidates if g % 4096 == 0 and fits(g)]
            if len(good) != 1:
                return None  # ambiguous or impossible: let the caller take the path that does not need file offsets
            base = good[0]
    except (RuntimeError, OSError):
        return None
    offs, end = [], 0
    for t in tensors:
        nb = t.numel() * t.element_size()
        off = t.data_ptr() - base if nb else -(-end // 16) * 16
        if off % 16 or off < end:
            return None
        offs.append(off)
        end = off + nb
    return offs


def patch_record_crcs(fd: int, records: Sequence[Tuple[str, int, int]], crcs: Sequence[int]) -> int:
    """Write the crc32 of data records into a container PyTorch laid out with ``torch.serialization.skip_data()`` (it leaves
    them zero: the data was not there to be summed).  ``records`` = ``(record name as the reader reports it, e.g. "data/7",
    data offset, size)``.  PyTorch's writer sets general-purpose flag bit 3, so a record's checksum lives in the data descriptor
    behind its data (signature 50 4b 07 08, then the crc) and in its central-directory entry; both are patched, the local header stays zero as
    PyTorch writes it.  Returns the number of records patched.  With this the file verifies (``zipfile.ZipFile.testzip()``)
    exactly like a file the reference's ``torch.save`` wrote (``async_ckpt/torch_ckpt.py:36-41``)."""
    want = {}
    for (name, off, size), crc in zip(records, crcs):
        want[name] = crc & _U32
        if os.pread(fd, 4, off + size) == b"PK\x07\x08":
            os.pwrite(fd, struct.pack("<I", crc & _U32), off + size + 4)
    end = os.fstat(fd).st_size
    tail_len = min(end, 65536 + 22 + 76)
    tail = os.pread(fd, tail_len, end - tail_len)
    eocd = tail.rfind(b"PK\x05\x06")
    if eocd < 0:
        raise ValueError("not a zip container: end-of-central-directory record not found")
    cd_size, cd_off = struct.unpack_from("<II", tail, eocd + 12)
    if cd_off == 0xFFFFFFFF or cd_size == 0xFFFFFFFF:
        loc = tail.rfind(b"PK\x06\x07", 0, eocd)
        if loc < 0:
            raise ValueError("zip64 locator missing")
        (z64_off,) = struct.unpack_from("<Q", tail, loc + 8)
        z64 = os.pread(fd, 56, z64_off)
        if z64[:4] != b"PK\x06\x06":
            raise ValueError("zip64 end-of-central-directory record missing")
        cd_size, cd_off = struct.unpack_from("<QQ", z64, 40)
    cd = bytearray(os.pread(fd, cd_size, cd_off))
    pos, patched = 0, 0
    while pos + 46 <= len(cd) and cd[pos:pos + 4] == b"PK\x01\x02":
        name_len, extra_len, comment_len = struct.unpack_from("<HHH", cd, pos + 28)
        name = bytes(cd[pos + 46:pos + 46 + name_len]).decode("utf-8", "replace")
        key = name.split("/", 1)[1] if "/" in name else name  # "<archive>/data/7" -> "data/7"
        if key in want:
            struct.pack_into("<I", cd, pos + 16, want[key])
            patched += 1
        pos += 46 + name_len + extra_len + comment_len
    os.pwrite(fd, bytes(cd), cd_off)
    return patched


def record_crcs(path, n_storages: int) -> Optional[List[int]]:
    """CRC-32 fields of the records ``data/0 .. data/n-1`` of a checkpoint file (from its central directory), or None when the
    file is not such an archive.  A zero field on a non-empty record means "written without checksums" (our fast writers'
    default; PyTorch's own writer and the GPU-checksum mode fill them in)."""
    import zipfile

    try:
        with zipfile.ZipFile(path) as zf:
            by_key = {k: info.CRC for k, info in _data_records(zf).items()}
    except (OSError, zipfile.BadZipFile):
        return None
    if sorted(by_key) != list(range(n_storages)):
        return None
    return [by_key[i] for i in range(n_storages)]


def _data_records(zf) -> dict:
    """``{k: ZipInfo}`` of the storage records ``<archive>/data/<k>`` of an open ``zipfile.ZipFile`` (zip64 included)."""
    by_key = {}
    for info in zf.infolist():
        head, sep, key = info.filename.rpartition("/data/")
        if sep and key.isdigit() and "/" not in head:
            by_key[int(key)] = info
    return by_key


class _FileWindow(io.RawIOBase):
    """Read-only, seekable view of ``[offset, offset + length)`` of an open file descriptor (positional reads only)."""

    def __init__(self, fd: int, offset: int, length: int):
        self._fd, self._off, self._len, self._pos = fd, offset, length, 0

    def readable(self):
        return True

    def seekable(self):
        return True

    def tell(self):
        return self._pos

    def seek(self, pos, whence=0):
        self._pos = {0: pos, 1: self._pos + pos, 2: self._len + pos}[whence]
        return self._pos

    def readinto(self, b):
        n = max(0, min(len(b), self._len - self._pos))
        data = os.pread(self._fd, n, self._off + self._pos) if n else b""
        b[: len(data)] = data
        self._pos += len(data)
        return len(data)


@dataclass
class SavedChunk:
    """What ``torch.load`` would rebuild from one embedded tensor archive, without its payload."""

    data_off: int  # file offset of the storage's first byte (the ``data/0`` record)
    dtype: torch.dtype
    numel: int  # elements of the storage
    storage_offset: int
    size: Tuple[int, ...]
    stride: Tuple[int, ...]
    crc32: int = 0  # the record's CRC-32 field in the central directory (0 on a non-empty record: written without one)
    record_len: int = 0  # byte length of the record (>= the storage's bytes)


class _TensorRecordUnpickler(pickle.Unpickler):
    """Reads the ``data.pkl`` of a single-tensor archive and executes nothing: only ``_rebuild_tensor_v2`` / ``_v3``, the
    typed-storage classes, ``torch.<dtype>`` and an empty ``OrderedDict`` (backward hooks) are known names, and all of them
    resolve to stand-ins that record their arguments."""

    _STORAGE_DTYPES = {name: dt for dt, name in torch.storage._dtype_to_storage_type_map().items()}

    def find_class(self, module, name):
        if module == "torch._utils" and name in ("_rebuild_tensor_v2", "_rebuild_tensor_v3"):
            return lambda storage, offset, size, stride, *rest: ("tensor", name, storage, offset, tuple(size), tuple(stride), rest)
        if module == "collections" and name == "OrderedDict":
            return lambda *a: ("hooks",) + a
        if module == "torch" and name in self._STORAGE_DTYPES:
            return ("typed", self._STORAGE_DTYPES[name])
        if module == "torch.storage" and name == "UntypedStorage":
            return ("typed", torch.uint8)
        if module == "torch" and isinstance(getattr(torch, name, None), torch.dtype):
            return ("dtype", getattr(torch, name))
        raise pickle.UnpicklingError(f"unexpected global {module}.{name} in a tensor record")

    def persistent_load(self, pid):
        if not (isinstance(pid, tuple) and len(pid) == 5 and pid[0] == "storage" and isinstance(pid[1], tuple)):
            raise pickle.UnpicklingError(f"unexpected persistent id {pid!r}")
        return ("storage", pid[1][1], str(pid[2]), int(pid[4]))


class RecordChecksumError(ValueError):
    """A member of a tensor archive whose bytes do not match its CRC-32 field (the same message zipfile gives)."""

    def __init__(self, member: str, header_off: int, got: int, expected: int):
        self.member, self.header_off, self.got, self.expected = member, header_off, got, expected
        super().__init__(f"not a single-tensor torch.save archive: Bad CRC-32 for file {member!r}")

    def __reduce__(self):  # picklable: torch.distributed.checkpoint gathers a rank's exception across ranks
        return type(self), (self.member, self.header_off, self.got, self.expected)


def _stored_payload(fd: int, offset: int, info) -> bytes:
    """The bytes of an uncompressed member ``info`` of the archive embedded at ``offset`` of ``fd``."""
    hdr = os.pread(fd, 30, offset + info.header_offset)
    if len(hdr) != 30 or hdr[:4] != b"PK\x03\x04":
        raise ValueError(f"bad local header of {info.filename}")
    name_len, extra_len = struct.unpack_from("<HH", hdr, 26)
    data = os.pread(fd, info.file_size, offset + info.header_offset + 30 + name_len + extra_len)
    if len(data) != info.file_size:
        raise ValueError(f"{info.filename} is truncated")
    return data


def read_tensor_record(fd: int, offset: int, length: int) -> SavedChunk:
    """Describe the ``torch.save`` archive of ONE tensor embedded at ``[offset, offset + length)`` of ``fd`` (how
    ``torch.distributed.checkpoint`` stores every tensor item of a ``.distcp`` file): where its payload starts, its dtype,
    element count, storage offset, size and stride (any strides: a chunk that was not cloned keeps them), and the storage
    record's CRC-32 field and byte length.  Reads the directory and ``data.pkl`` only -- not the payload -- and never runs
    code from the pickle; ``ValueError`` when the window is not such an archive, ``RecordChecksumError`` (a ValueError)
    when ``data.pkl`` does not match its non-zero CRC-32 field."""
    import zipfile

    try:
        with zipfile.ZipFile(_FileWindow(fd, offset, length)) as zf:
            recs = _data_records(zf)
            pkl = [i for i in zf.infolist() if i.filename.endswith("/data.pkl") and i.filename.count("/") == 1]
            if len(pkl) != 1:
                raise ValueError("no data.pkl record")
            # read the stored pickle directly and check it against its CRC-32 field like zipfile does, except when the field
            # is 0: an archive written with torch.serialization.set_crc32_options(False) (torch.load accepts those)
            pkl_bytes = _stored_payload(fd, offset, pkl[0]) if pkl[0].compress_type == zipfile.ZIP_STORED else zf.read(pkl[0])
            if pkl[0].CRC and zlib.crc32(pkl_bytes) != pkl[0].CRC:
                raise RecordChecksumError(pkl[0].filename, offset + pkl[0].header_offset, zlib.crc32(pkl_bytes), pkl[0].CRC)
            rec = _TensorRecordUnpickler(io.BytesIO(pkl_bytes)).load()
            if not (isinstance(rec, tuple) and rec[0] == "tensor" and rec[2][0] == "storage"):
                raise ValueError("data.pkl does not describe a single tensor")
            _, fn, (_, st_dtype, key, st_numel), st_off, size, stride, rest = rec
            dtype = st_dtype
            if fn == "_rebuild_tensor_v3":
                dts = [r[1] for r in rest if isinstance(r, tuple) and r and r[0] == "dtype"]
                if len(dts) != 1:
                    raise ValueError("_rebuild_tensor_v3 record without a dtype")
                dtype = dts[0]
                elem = torch.empty(0, dtype=dtype).element_size()
                st_numel //= elem  # an untyped storage counts bytes
            if not key.isdigit() or int(key) not in recs:
                raise ValueError(f"storage record data/{key} missing")
            info = recs[int(key)]
            if info.file_size < st_numel * torch.empty(0, dtype=dtype).element_size():
                raise ValueError("storage record shorter than its storage")
            if info.compress_type != zipfile.ZIP_STORED:
                raise ValueError("compressed storage record")
            hdr = os.pread(fd, 30, offset + info.header_offset)
            if len(hdr) != 30 or hdr[:4] != b"PK\x03\x04":
                raise ValueError("bad local header of the storage record")
            name_len, extra_len = struct.unpack_from("<HH", hdr, 26)
            data_off = offset + info.header_offset + 30 + name_len + extra_len
    except (zipfile.BadZipFile, pickle.UnpicklingError, EOFError, TypeError, IndexError) as e:
        raise ValueError(f"not a single-tensor torch.save archive: {e}") from e
    return SavedChunk(data_off=data_off, dtype=dtype, numel=int(st_numel), storage_offset=int(st_off), size=size, stride=stride,
                      crc32=int(info.CRC), record_len=int(info.file_size))
