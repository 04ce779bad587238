"""Host side of the H100 snapshot engine: thin objects over the C ABI plus the snapshot pipeline.

Pipeline of one snapshot (``SnapshotEngine.snapshot``)::

    tensors (HBM) --nvrx_pack (1 kernel, current stream)--> staging (HBM)
                  --nvrx_drain (cudaMemcpyAsync, side stream)--> HostBuffer (pinned POSIX shm)
                  --CPU-only writer process follows HostBuffer.progress--> file

What it replaces in the reference (paths relative to ``src/nvidia_resiliency_ext/checkpointing``):

* ``utils.py:85-99`` ``preload_tensors`` and ``local/basic_state_dict.py:162-174`` ``copy_tensors_to_cpu``:
  N x (pinned allocation + ``cudaMemcpyAsync`` D2H) on the training stream, followed by a device-wide
  ``torch.cuda.synchronize()`` (``async_ckpt/torch_ckpt.py:50``, ``local/ckpt_managers/base_manager.py:306-309``).
  Here the training stream only carries the pack kernel; the D2H runs on a side stream.
* ``local/basic_state_dict.py:176-187`` ``restore_tensor_device``: N blocking H2D copies -> one H2D + one
  scatter kernel (``SnapshotEngine.restore``).

There is no CPU fallback: everything here raises if ``libnvrx_snap.so`` or a CUDA device is missing.
"""

from __future__ import annotations

import ctypes as C
import logging
import os
import re
import threading
import uuid
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence, Tuple

import torch

from . import _cabi
from ._cabi import SnapError, check

logger = logging.getLogger(__name__)

DEFAULT_ALIGN = 512
DEFAULT_DRAIN_CHUNK = int(os.environ.get("NVRX_B200_DRAIN_CHUNK_MB", "256")) << 20


def _ptr_array(values: Sequence[int]):
    arr = (C.c_void_p * max(len(values), 1))()
    for i, v in enumerate(values):
        arr[i] = v
    return arr


def _u64_array(values: Sequence[int]):
    return (C.c_uint64 * max(len(values), 1))(*values)


def _u32_array(values: Sequence[int]):
    return (C.c_uint32 * max(len(values), 1))(*values)


class Plan:
    """A compiled tensor table (``nvrx_plan``): segment layout in staging + tile work-list on the device."""

    def __init__(
        self,
        ptrs: Sequence[int],
        nbytes: Sequence[int],
        flags: Optional[Sequence[int]] = None,
        *,
        device: int,
        align: int = 0,
        tile_bytes: int = 0,
        variant: int = _cabi.VARIANT_AUTO,
        staging_offsets: Optional[Sequence[int]] = None,
    ):
        assert len(ptrs) == len(nbytes)
        self._lib = _cabi.lib()
        self.n = len(ptrs)
        self.device = device
        self._h = C.c_void_p()
        flags_arr = _u32_array(flags) if flags is not None else None
        offs_arr = _u64_array(staging_offsets) if staging_offsets is not None else None
        check(
            self._lib.nvrx_plan_create_at(
                self.n, _ptr_array(ptrs), _u64_array(nbytes), flags_arr, offs_arr, align, tile_bytes, device, C.byref(self._h)
            ),
            "nvrx_plan_create_at",
        )
        stg, tiles, algo = C.c_uint64(), C.c_uint64(), C.c_uint64()
        check(self._lib.nvrx_plan_info(self._h, C.byref(stg), C.byref(tiles), C.byref(algo)), "nvrx_plan_info")
        self.staging_bytes = stg.value
        self.algorithmic_bytes = algo.value
        offs, packed = _u64_array([0] * self.n), _u64_array([0] * self.n)
        check(self._lib.nvrx_plan_layout(self._h, offs, packed), "nvrx_plan_layout")
        self.offsets: Tuple[int, ...] = tuple(offs[i] for i in range(self.n))
        self.packed_nbytes: Tuple[int, ...] = tuple(packed[i] for i in range(self.n))
        self.ptrs: Tuple[int, ...] = tuple(ptrs)
        if variant != _cabi.VARIANT_AUTO:
            self.set_variant(variant)

    @property
    def n_tiles(self) -> int:
        tiles = C.c_uint64()
        check(self._lib.nvrx_plan_info(self._h, None, C.byref(tiles), None), "nvrx_plan_info")
        return tiles.value

    def tiles(self, shard_bytes: int = 0):
        """(n_bulk, [(seg, nbytes, off), ...]) -- the work-list as the kernels would walk it (no CUDA involved)."""
        nb, nt = C.c_uint32(), C.c_uint32()
        check(self._lib.nvrx_plan_tiles(self._h, shard_bytes, C.byref(nb), C.byref(nt), None, None, None, 0), "nvrx_plan_tiles")
        n = nt.value
        seg, nby, off = (C.c_uint32 * max(n, 1))(), (C.c_uint32 * max(n, 1))(), (C.c_uint64 * max(n, 1))()
        check(self._lib.nvrx_plan_tiles(self._h, shard_bytes, C.byref(nb), C.byref(nt), seg, nby, off, n), "nvrx_plan_tiles")
        return nb.value, [(seg[i], nby[i], off[i]) for i in range(n)]

    def last_launches(self) -> int:
        n = C.c_uint32()
        check(self._lib.nvrx_plan_last_launches(self._h, C.byref(n)), "nvrx_plan_last_launches")
        return n.value

    def set_variant(self, variant: int) -> None:
        check(self._lib.nvrx_plan_set_variant(self._h, variant), "nvrx_plan_set_variant")

    def update_ptrs(self, ptrs: Sequence[int]) -> None:
        assert len(ptrs) == self.n
        if tuple(ptrs) == self.ptrs:
            return
        check(self._lib.nvrx_plan_update_ptrs(self._h, _ptr_array(ptrs)), "nvrx_plan_update_ptrs")
        self.ptrs = tuple(ptrs)

    def commit(self, stream: int) -> None:
        check(self._lib.nvrx_plan_commit(self._h, stream), "nvrx_plan_commit")

    def pack(self, staging_ptr: int, stream: int) -> None:
        check(self._lib.nvrx_pack(self._h, staging_ptr, stream), "nvrx_pack")

    def scatter(self, staging_ptr: int, stream: int) -> None:
        check(self._lib.nvrx_scatter(self._h, staging_ptr, stream), "nvrx_scatter")

    def pack_sharded(self, staging_ptr: Optional[int], peer_bases: Sequence[int], shard_bytes: int, slot_offset: int, stream: int) -> None:
        check(
            self._lib.nvrx_pack_sharded(
                self._h, staging_ptr, _ptr_array(peer_bases), len(peer_bases), shard_bytes, slot_offset, stream
            ),
            "nvrx_pack_sharded",
        )

    def set_shard_rotation(self, first_shard: int) -> None:
        check(self._lib.nvrx_plan_set_shard_rotation(self._h, first_shard), "nvrx_plan_set_shard_rotation")

    def pack_broadcast(self, peer_bases: Sequence[int], slot_offset: int, stream: int) -> None:
        check(
            self._lib.nvrx_pack_broadcast(self._h, _ptr_array(peer_bases), len(peer_bases), slot_offset, stream),
            "nvrx_pack_broadcast",
        )

    def close(self) -> None:
        if self._h:
            self._lib.nvrx_plan_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class DeviceBuffer:
    """cudaMalloc'ed, zero-filled, IPC-exportable device memory (``nvrx_dev_alloc``)."""

    def __init__(self, nbytes: int, device: int):
        self._lib = _cabi.lib()
        self.device = device
        self.nbytes = nbytes
        p = C.c_void_p()
        check(self._lib.nvrx_dev_alloc(device, nbytes, C.byref(p)), "nvrx_dev_alloc")
        self.ptr = p.value

    def ipc_handle(self) -> bytes:
        buf = C.create_string_buffer(64)
        check(self._lib.nvrx_ipc_export(self.ptr, buf), "nvrx_ipc_export")
        return buf.raw

    def close(self) -> None:
        if self.ptr:
            self._lib.nvrx_dev_free(self.device, self.ptr)
            self.ptr = 0

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class Stream:
    def __init__(self, device: int, high_priority: bool = False):
        self._lib = _cabi.lib()
        p = C.c_void_p()
        check(self._lib.nvrx_stream_create(device, int(high_priority), C.byref(p)), "nvrx_stream_create")
        self.handle = p.value

    def synchronize(self) -> None:
        check(self._lib.nvrx_stream_sync(self.handle), "nvrx_stream_sync")

    def wait_event(self, ev: "Event") -> None:
        check(self._lib.nvrx_stream_wait_event(self.handle, ev.handle), "nvrx_stream_wait_event")

    def close(self) -> None:
        if self.handle:
            self._lib.nvrx_stream_destroy(self.handle)
            self.handle = 0

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class Event:
    def __init__(self, device: int, timing: bool = False):
        self._lib = _cabi.lib()
        p = C.c_void_p()
        check(self._lib.nvrx_event_create(device, int(timing), C.byref(p)), "nvrx_event_create")
        self.handle = p.value

    def record(self, stream: int) -> None:
        check(self._lib.nvrx_event_record(self.handle, stream), "nvrx_event_record")

    def query(self) -> bool:
        done = C.c_int()
        check(self._lib.nvrx_event_query(self.handle, C.byref(done)), "nvrx_event_query")
        return bool(done.value)

    def synchronize(self) -> None:
        check(self._lib.nvrx_event_sync(self.handle), "nvrx_event_sync")

    def elapsed_ms(self, end: "Event") -> float:
        ms = C.c_float()
        check(self._lib.nvrx_event_elapsed_ms(self.handle, end.handle, C.byref(ms)), "nvrx_event_elapsed_ms")
        return ms.value

    def close(self) -> None:
        if self.handle:
            self._lib.nvrx_event_destroy(self.handle)
            self.handle = 0

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class CrcPlan:
    """Extents of a packed device buffer whose zlib CRC-32s the GPU computes (``nvrx_crc_*``).  Creating it is CUDA-free."""

    def __init__(self, offsets: Sequence[int], nbytes: Sequence[int], device: int):
        self._lib = _cabi.lib()
        self._h = C.c_void_p()
        n = len(offsets)
        check(self._lib.nvrx_crc_create(n, _u64_array(offsets), _u64_array(nbytes), device, C.byref(self._h)), "nvrx_crc_create")
        cnt = C.c_uint64()
        check(self._lib.nvrx_crc_info(self._h, C.byref(cnt)), "nvrx_crc_info")
        self.n_values = cnt.value

    def run(self, dev_base: int, host_values: int, host_ready: int, ready_value: int, stream: int) -> None:
        check(self._lib.nvrx_crc_run(self._h, dev_base, host_values, host_ready, ready_value, stream), "nvrx_crc_run")

    def close(self) -> None:
        if self._h:
            self._lib.nvrx_crc_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def finish_crcs(offsets: Sequence[int], nbytes: Sequence[int], values_ptr: int, n_values: int, host_base: int) -> List[int]:
    """CPU only: crc32 of every extent from the GPU's partial values and the host copy of the buffer (``nvrx_crc_finish``)."""
    n = len(offsets)
    out = (C.c_uint32 * max(n, 1))()
    check(
        _cabi.lib().nvrx_crc_finish(n, _u64_array(offsets), _u64_array(nbytes), values_ptr, n_values, host_base, out),
        "nvrx_crc_finish",
    )
    return [out[i] for i in range(n)]


def gpu_crc_enabled() -> bool:
    """Opt-in (``NVRX_B200_GPU_CRC=1``): record checksums of checkpoint files come from a kernel over the staging buffer
    instead of from the writer's CPU threads (the default: ``nvrx_hostbuf_crc32v``, PCLMULQDQ folding; ``NVRX_B200_ZIP_CRC=0``
    leaves them zero)."""
    return os.environ.get("NVRX_B200_GPU_CRC", "0") == "1"


def stream_wait_event(stream: int, ev: Event) -> None:
    check(_cabi.lib().nvrx_stream_wait_event(stream, ev.handle), "nvrx_stream_wait_event")


class HostBuffer:
    """One snapshot slot in host memory: a POSIX shm mapping with a progress word, optionally pinned."""

    def __init__(self, handle: int, name: Optional[str], owner: bool):
        self._lib = _cabi.lib()
        self._h = C.c_void_p(handle)
        self.name = name
        self.owner = owner
        self.data_ptr: int = self._lib.nvrx_hostbuf_data(self._h)
        self.capacity: int = self._lib.nvrx_hostbuf_capacity(self._h)
        self.progress_ptr: int = self._lib.nvrx_hostbuf_progress(self._h)

    @classmethod
    def create(
        cls, nbytes: int, *, name: Optional[str] = None, pin: bool = True, device: int = 0, prefault_threads: int = 0
    ) -> "HostBuffer":
        h = C.c_void_p()
        cname = name.encode() if name else None
        check(
            _cabi.lib().nvrx_hostbuf_create(cname, nbytes, prefault_threads, int(pin), device, C.byref(h)),
            "nvrx_hostbuf_create",
        )
        return cls(h.value, name, owner=True)

    @classmethod
    def open(cls, name: str) -> "HostBuffer":
        h = C.c_void_p()
        check(_cabi.lib().nvrx_hostbuf_open(name.encode(), C.byref(h)), "nvrx_hostbuf_open")
        return cls(h.value, name, owner=False)

    @property
    def progress(self) -> int:
        return C.c_uint64.from_address(self.progress_ptr).value

    def wait(self, value: int, timeout_ms: int = -1) -> None:
        check(self._lib.nvrx_hostbuf_wait(self._h, value, timeout_ms), "nvrx_hostbuf_wait")

    def as_tensor(self, nbytes: Optional[int] = None) -> torch.Tensor:
        """uint8 tensor over the first ``nbytes`` of the payload (default: all of it), no copy.

        The tensor's *storage* is exactly ``nbytes`` long, so ``torch.save`` of views into it writes the
        snapshot and not the slot's spare capacity.  The mapping must outlive the tensor."""
        nbytes = self.capacity if nbytes is None else nbytes
        assert 0 <= nbytes <= self.capacity
        if nbytes == 0:
            return torch.empty(0, dtype=torch.uint8)
        raw = (C.c_uint8 * nbytes).from_address(self.data_ptr)
        return torch.frombuffer(raw, dtype=torch.uint8)

    def segment(self, offset: int, nbytes: int, dtype: torch.dtype, shape) -> torch.Tensor:
        """Typed CPU tensor over ``[offset, offset + nbytes)`` of the payload with a *storage of its own*.

        ``torch.save`` refuses tensors of different dtypes that share one storage, and would write the whole
        slot for every view; one storage per segment gives the same file structure as the reference's
        per-tensor host copies (one record per tensor) without copying anything."""
        assert 0 <= offset and offset + nbytes <= self.capacity
        if nbytes == 0:
            return torch.empty(shape, dtype=dtype)
        raw = (C.c_uint8 * nbytes).from_address(self.data_ptr + offset)
        t = torch.frombuffer(raw, dtype=dtype).view(shape)
        return t

    def write_fd(self, offset: int, nbytes: int, fd: int, file_off: int, threads: int = 8) -> None:
        check(self._lib.nvrx_hostbuf_write_fd(self._h, offset, nbytes, fd, file_off, threads), "nvrx_hostbuf_write_fd")

    def writev_fd(self, offsets: Sequence[int], nbytes: Sequence[int], file_offs: Sequence[int], fd: int, threads: int = 8) -> None:
        n = len(offsets)
        check(
            self._lib.nvrx_hostbuf_writev_fd(self._h, n, _u64_array(offsets), _u64_array(nbytes), _u64_array(file_offs), fd, threads),
            "nvrx_hostbuf_writev_fd",
        )

    def readv_fd(self, offsets: Sequence[int], nbytes: Sequence[int], file_offs: Sequence[int], fd: int, threads: int = 16) -> None:
        n = len(offsets)
        check(
            self._lib.nvrx_hostbuf_readv_fd(self._h, n, _u64_array(offsets), _u64_array(nbytes), _u64_array(file_offs), fd, threads),
            "nvrx_hostbuf_readv_fd",
        )

    def gather(self, src_ptrs: Sequence[int], nbytes: Sequence[int], dst_offsets: Sequence[int], threads: int = 16) -> None:
        check(
            self._lib.nvrx_hostbuf_gather(self._h, len(src_ptrs), _ptr_array(src_ptrs), _u64_array(nbytes), _u64_array(dst_offsets), threads),
            "nvrx_hostbuf_gather",
        )

    def crc32(self, offset: int, nbytes: int, threads: int = 8) -> int:
        out = C.c_uint32()
        check(self._lib.nvrx_hostbuf_crc32(self._h, offset, nbytes, threads, C.byref(out)), "nvrx_hostbuf_crc32")
        return out.value

    def crc32v(self, offsets: Sequence[int], nbytes: Sequence[int], threads: int = 16) -> List[int]:
        """zlib crc32 of every extent ``[offsets[i], +nbytes[i])`` of the payload, one threaded pass."""
        n = len(offsets)
        out = (C.c_uint32 * max(n, 1))()
        check(self._lib.nvrx_hostbuf_crc32v(self._h, n, _u64_array(offsets), _u64_array(nbytes), threads, out), "nvrx_hostbuf_crc32v")
        return [out[i] for i in range(n)]

    def close(self, unlink: Optional[bool] = None) -> None:
        if self._h:
            self._lib.nvrx_hostbuf_destroy(self._h, int(self.owner if unlink is None else unlink))
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


# --------------------------------------------------------------------------------------------------
# layout description that travels to writer processes / into checkpoint files
# --------------------------------------------------------------------------------------------------
_DTYPE_NAMES = {
    str(d).replace("torch.", ""): d
    for d in (
        torch.float32, torch.float64, torch.float16, torch.bfloat16, torch.int8, torch.uint8, torch.int16,
        torch.int32, torch.int64, torch.bool, torch.complex64, torch.complex128,
    )
}
for _extra in ("float8_e4m3fn", "float8_e5m2", "uint16", "uint32", "uint64"):
    if hasattr(torch, _extra):
        _DTYPE_NAMES[_extra] = getattr(torch, _extra)


def dtype_name(dtype: torch.dtype) -> str:
    return str(dtype).replace("torch.", "")


@dataclass
class PackedLayout:
    """Where every tensor of a flattened state dict lives inside a packed buffer."""

    shapes: List[Tuple[int, ...]]
    dtypes: List[str]  # dtype of the *packed* data (bf16 for narrowed fp32 tensors)
    src_dtypes: List[str]  # dtype of the tensor on the device
    offsets: List[int]
    packed_nbytes: List[int]
    total_bytes: int
    align: int = DEFAULT_ALIGN

    def views(self, buf: torch.Tensor) -> List[torch.Tensor]:
        """Typed tensor views into a uint8 buffer holding the packed bytes."""
        out = []
        for shape, dt, off, nb in zip(self.shapes, self.dtypes, self.offsets, self.packed_nbytes):
            dtype = _DTYPE_NAMES[dt]
            if nb == 0:
                out.append(torch.empty(shape, dtype=dtype, device=buf.device))
            else:
                out.append(buf[off : off + nb].view(dtype).view(shape))
        return out


def host_views(layout: "PackedLayout", hb: "HostBuffer") -> List[torch.Tensor]:
    """One CPU tensor per segment of ``layout`` inside host buffer ``hb`` (each with its own storage)."""
    return [
        hb.segment(off, nb, _DTYPE_NAMES[dt], shape)
        for shape, dt, off, nb in zip(layout.shapes, layout.dtypes, layout.offsets, layout.packed_nbytes)
    ]


def expected_layout(nbytes: Sequence[int], narrow: Sequence[bool], align: int = DEFAULT_ALIGN) -> Tuple[List[int], List[int], int]:
    """Pure-Python statement of the layout rule in include/nvrx_snap.h (used for cross-checks only)."""
    offs, packed, cur = [], [], 0
    for nb, nr in zip(nbytes, narrow):
        cur = (cur + align - 1) // align * align
        offs.append(cur)
        pk = nb // 2 if nr else nb
        packed.append(pk)
        cur += pk
    return offs, packed, (cur + align - 1) // align * align


# --------------------------------------------------------------------------------------------------
# the pipeline
# --------------------------------------------------------------------------------------------------
@dataclass
class _Slot:
    index: int
    buf: Optional[HostBuffer] = None
    busy: bool = False
    drained_total: int = 0  # cumulative bytes the progress word has been advanced by
    done_event: Optional[Event] = None

    def published(self) -> bool:
        """A checkpoint file is a hard link to this slot (zero-copy persistence): its pages must not be overwritten."""
        if self.buf is None or not self.buf.name:
            return False
        from .ptzip import slot_is_published

        return slot_is_published("/dev/shm" + self.buf.name)


@dataclass
class Snapshot:
    """Handle of one in-flight / completed snapshot."""

    engine: "SnapshotEngine"
    slot: _Slot
    layout: PackedLayout
    progress_target: int
    passthrough: Dict[int, torch.Tensor] = field(default_factory=dict)  # position -> non-CUDA tensor kept as is
    n_total: int = 0
    pack_start: Optional[Event] = None
    pack_stop: Optional[Event] = None
    released: bool = False
    crc_info: Optional[dict] = None  # where the GPU's checksum values land in the slot (opt-in, see gpu_crc_enabled)

    def drained(self) -> bool:
        return self.slot.done_event.query()

    def wait(self) -> None:
        """Block the calling CPU thread until the bytes are in host memory (no device-wide sync)."""
        self.slot.done_event.synchronize()

    def host_views(self) -> List[torch.Tensor]:
        """CPU tensor views (one per input tensor, input order) into the pinned shm slot.

        Their *content* is valid once :meth:`wait` returned / ``drained()`` is true -- same contract as the
        reference's ``tensor.to("cpu", non_blocking=True)`` before ``torch.cuda.synchronize()``."""
        packed = host_views(self.layout, self.slot.buf)
        if not self.passthrough:
            return packed
        out, it = [], iter(packed)
        for i in range(self.n_total):
            out.append(self.passthrough[i] if i in self.passthrough else next(it))
        return out

    def pack_ms(self) -> float:
        self.pack_stop.synchronize()
        return self.pack_start.elapsed_ms(self.pack_stop)

    def descriptor(self) -> dict:
        """Picklable description a CPU-only process needs to follow and read this snapshot."""
        return {
            "shm_name": self.slot.buf.name,
            "progress_target": self.progress_target,
            "layout": self.layout,
            "owner_pid": os.getpid(),
            "owner_base": self.slot.buf.data_ptr,  # where the trainer's views of the slot live (valid in fork children)
            "crc": self.crc_info,
        }

    def release(self) -> None:
        if not self.released:
            self.released = True
            self.engine._release(self.slot)


def choose_slot(slots: Sequence[_Slot], nbytes: int, max_slots: int) -> Tuple[Optional[_Slot], bool]:
    """Which slot the next snapshot of ``nbytes`` goes to: ``(slot, retire)``.

    Prefer an idle slot that is already large enough (no re-pinning), then any idle slot.  A slot that was published as a
    checkpoint file (hard link, zero-copy persistence) is idle again once that file has been deleted; while the file exists
    it is skipped.  ``(None, False)`` = grow the pool if allowed; ``retire`` = the pool is at its bound and every idle slot
    is a checkpoint somebody keeps, so one of them has to be given up to the file system."""
    idle = [s for s in slots if not s.busy]
    free = [s for s in idle if not s.published()]
    pick = next((s for s in free if s.buf is not None and s.buf.capacity >= nbytes), free[0] if free else None)
    if pick is None and len(slots) >= max_slots:
        kept = next((s for s in idle if s.published()), None)
        if kept is not None:
            return kept, True
    return pick, False


_SLOT_NAME = re.compile(r"^nvrx_b200_(\d+)_(\d+)_[0-9a-f]{8}_s\d+_g\d+$")
_reaped = False


def _pid_namespace() -> int:
    try:
        return os.stat("/proc/self/ns/pid").st_ino
    except OSError:
        return 0


def reap_stale_slots(shm_dir: str = "/dev/shm") -> List[str]:
    """Remove snapshot slots whose owner died without running its exit handler (SIGKILL, OOM kill, node-local crash): each is
    a shared-memory object as large as a snapshot and would otherwise stay until reboot, counting against the container's
    memory.  A slot belongs to a dead owner when its name carries this PID namespace and a PID that no longer exists.  Only
    the shm NAME is removed: a checkpoint file that is a hard link to the slot (zero-copy persistence) keeps its pages, which is
    the point of a local checkpoint.  Returns the names removed."""
    removed = []
    ns = _pid_namespace()
    try:
        names = os.listdir(shm_dir)
    except OSError:
        return removed
    for name in names:
        m = _SLOT_NAME.match(name)
        if not m or int(m.group(1)) != ns:
            continue
        pid = int(m.group(2))
        try:
            os.kill(pid, 0)
            continue  # alive (or not ours to signal: PermissionError below)
        except ProcessLookupError:
            pass
        except OSError:
            continue
        try:
            os.unlink(os.path.join(shm_dir, name))
            removed.append(name)
        except OSError:
            pass
    return removed


def spare_slots(slots: Sequence[_Slot], max_slots: int) -> int:
    return sum(1 for s in slots if not s.busy and not s.published()) + max(0, max_slots - len(slots))


class SnapshotEngine:
    """Per-(process, device) snapshot engine.  Thread-compatible: call from the training thread."""

    _instances: Dict[int, "SnapshotEngine"] = {}
    _lock = threading.Lock()

    def __init__(
        self,
        device: Optional[int] = None,
        *,
        host_slots: int = 2,
        align: int = DEFAULT_ALIGN,
        tile_bytes: int = 0,
        variant: Optional[int] = None,
        drain_chunk: int = DEFAULT_DRAIN_CHUNK,
        shm_prefix: Optional[str] = None,
        timing: bool = False,
        prefault_threads: Optional[int] = None,
    ):
        if not torch.cuda.is_available():
            raise SnapError(_cabi.E_STATE, "SnapshotEngine", "no CUDA device - the snapshot path has no CPU fallback")
        self.lib = _cabi.lib()
        self.device = torch.cuda.current_device() if device is None else int(device)
        self.align = align
        self.tile_bytes = tile_bytes or int(os.environ.get("NVRX_B200_TILE_BYTES", "0"))
        if variant is None:
            variant = {"auto": 0, "ldg": 1, "tma": 2}[os.environ.get("NVRX_B200_VARIANT", "auto").lower()]
        self.variant = variant
        self.drain_chunk = drain_chunk
        self.timing = timing
        self.prefault_threads = prefault_threads if prefault_threads is not None else min(16, os.cpu_count() or 1)
        self.shm_prefix = shm_prefix or f"/nvrx_b200_{_pid_namespace()}_{os.getpid()}_{uuid.uuid4().hex[:8]}"
        global _reaped
        if not _reaped and os.environ.get("NVRX_B200_NO_REAP", "0") != "1":
            _reaped = True
            stale = reap_stale_slots()
            if stale:
                logger.warning(f"removed {len(stale)} snapshot slot(s) left behind by dead processes: {stale[:4]}...")
        self._plans: Dict[tuple, Plan] = {}
        self._staging: Optional[DeviceBuffer] = None
        self._staging_free: Optional[Event] = None  # recorded when the last reader of staging finished
        self._side = Stream(self.device)
        self._slots = [_Slot(i) for i in range(max(1, host_slots))]
        self.max_host_slots = max(len(self._slots), int(os.environ.get("NVRX_B200_MAX_HOST_SLOTS", "4")))
        self._slot_gen = 0
        self.launches = 0  # kernels launched by this engine (pack + scatter)
        self.resident_restores = 0  # restores that read a published slot in place (no host copy)
        self.file_restores = 0  # restores fed straight from the checkpoint file through the pinned ring
        self._aux: Optional[Stream] = None  # checksum kernels (created on first use)
        self._pid = os.getpid()  # forked writers inherit this object; only the creator may tear it down
        # NVRX_B200_TRACE=1: host-side time stamps of the last snapshot() (enter / planned / launched), for the stall breakdown
        self.trace: Optional[dict] = {} if os.environ.get("NVRX_B200_TRACE", "0") == "1" else None

    # ---- singletons per device ------------------------------------------------------------------
    @classmethod
    def get(cls, device: Optional[int] = None, **kwargs) -> "SnapshotEngine":
        dev = torch.cuda.current_device() if device is None else int(device)
        with cls._lock:
            eng = cls._instances.get(dev)
            if eng is None:
                eng = cls(dev, **kwargs)
                cls._instances[dev] = eng
            return eng

    @classmethod
    def shutdown_all(cls) -> None:
        with cls._lock:
            for eng in cls._instances.values():
                eng.close()
            cls._instances.clear()

    # ---- resources ------------------------------------------------------------------------------
    def _current_stream(self) -> int:
        return torch.cuda.current_stream(self.device).cuda_stream

    def _ensure_staging(self, nbytes: int) -> DeviceBuffer:
        if self._staging is None or self._staging.nbytes < nbytes:
            if self._staging is not None:
                if self._staging_free is not None:
                    self._staging_free.synchronize()
                self._staging.close()
            self._staging = DeviceBuffer(max(nbytes, 512), self.device)
        return self._staging

    def _acquire_slot(self, nbytes: int, slot: Optional[_Slot] = None) -> _Slot:
        if slot is None:
            slot, retire = choose_slot(self._slots, nbytes, self.max_host_slots)
            if retire:
                # the pool is full of checkpoints somebody keeps: give this one up (the file keeps the pages, this process
                # drops its mapping and pinning) and start a fresh buffer in its place
                slot.__dict__.pop("_exchange_views", None)
                slot.buf.close()
                slot.buf = None
        if slot is None and len(self._slots) < self.max_host_slots:
            # every slot still belongs to an unfinalized save: grow the pool (the reference allocates fresh pinned
            # memory for every save, too); bounded so a caller that never finalizes fails loudly instead of eating RAM
            slot = _Slot(len(self._slots))
            self._slots.append(slot)
        if slot is None:
            raise SnapError(
                _cabi.E_STATE,
                "acquiring a host snapshot slot",
                f"all {len(self._slots)} slots hold unfinalized snapshots; finalize earlier saves first "
                "(or raise NVRX_B200_MAX_HOST_SLOTS)",
            )
        if slot.buf is None or slot.buf.capacity < nbytes:
            slot.__dict__.pop("_exchange_views", None)  # cached host views of the old buffer (b200/exchange.py)
            if slot.buf is not None:
                slot.buf.close()
            self._slot_gen += 1
            name = f"{self.shm_prefix}_s{slot.index}_g{self._slot_gen}"
            slot.buf = HostBuffer.create(
                nbytes, name=name, pin=True, device=self.device, prefault_threads=self.prefault_threads
            )
            slot.drained_total = 0
        if slot.done_event is None:
            slot.done_event = Event(self.device)
        slot.busy = True
        return slot

    def _release(self, slot: _Slot) -> None:
        slot.busy = False

    def _spare_slots(self) -> int:
        """Slots a snapshot could go to without giving up a published checkpoint: idle unpublished ones plus pool headroom."""
        return spare_slots(self._slots, self.max_host_slots)

    def reserve(self, nbytes: int, n_tensors: int = 0) -> None:
        """Pre-allocate staging and every host slot for snapshots of up to ``nbytes`` packed bytes of ``n_tensors``
        tensors (pinning 16 GB takes seconds; do it once at start-up instead of inside the first save).  With zero-copy
        persistence on, a slot also holds the checkpoint file's small records and directory behind the payload: that
        room is reserved too, or the first save would re-create and re-pin the slot."""
        from .fastsave import zero_copy_enabled
        from .ptzip import slot_tail_room

        self._ensure_staging(nbytes)
        slot_bytes = nbytes + (slot_tail_room(n_tensors) if zero_copy_enabled() else 0)
        for s in self._slots:
            if not s.busy and not s.published():
                self._acquire_slot(slot_bytes, s)
                self._release(s)

    # ---- planning -------------------------------------------------------------------------------
    def _plan_for(
        self, tensors: Sequence[torch.Tensor], narrow: Sequence[bool], container: bool = False,
        offsets: Optional[Sequence[int]] = None,
    ) -> Plan:
        """Cached plan for tensors of these sizes/dtypes.  ``container``: staging offsets follow the checkpoint-container
        geometry of ``ptzip.slot_offsets`` (room for a ZIP local header in front of every segment) instead of the dense
        default, so that the drained slot can be published as a file without a copy.  ``offsets``: explicit staging
        offsets (restore straight from a published slot)."""
        nbytes = [t.nbytes for t in tensors]
        if narrow is not None and not any(narrow):
            narrow = None
        # a bit copy does not care about dtypes (the layout handed to readers does: it is validated where it is cached)
        key = (tuple(nbytes), tuple(narrow) if narrow is not None else None)
        if offsets is not None:
            key = ("at", tuple(offsets)) + key
        elif container:
            key = ("container",) + key
        ptrs = [t.data_ptr() if nb else 0 for t, nb in zip(tensors, nbytes)]
        plan = self._plans.get(key)
        if plan is None:
            if narrow is None:
                narrow = [False] * len(tensors)
            flags = [_cabi.SEG_NARROW_F32_BF16 if nr else 0 for nr in narrow]
            if offsets is None and container:
                from .ptzip import slot_offsets

                offsets, _ = slot_offsets([nb // 2 if nr else nb for nb, nr in zip(nbytes, narrow)])
            plan = Plan(
                ptrs, nbytes, flags, device=self.device, align=self.align, tile_bytes=self.tile_bytes,
                variant=self.variant, staging_offsets=offsets,
            )
            self._plans[key] = plan
        else:
            plan.update_ptrs(ptrs)
        return plan

    @staticmethod
    def _narrow_mask(tensors: Sequence[torch.Tensor], narrow: bool) -> List[bool]:
        return [bool(narrow) and t.dtype == torch.float32 and t.numel() > 0 for t in tensors]

    # ---- snapshot -------------------------------------------------------------------------------
    def snapshot(self, tensors: Sequence[torch.Tensor], *, narrow: bool = False, container: Optional[bool] = None) -> Snapshot:
        """Pack ``tensors`` (CUDA tensors of this device; others pass through) and start the drain.

        Returns as soon as the pack kernel and the side-stream copy are *enqueued*.  ``container`` (default: the
        ``NVRX_B200_ZERO_COPY`` switch) packs in checkpoint-container geometry, see :meth:`_plan_for`."""
        trace = self.trace
        if trace is not None:
            import time as _time

            trace.clear()
            trace["enter"] = _time.perf_counter()
        all_tensors = tensors if isinstance(tensors, list) else list(tensors)
        dev = self.device
        # everything up to the launch is on the training stream's critical path (the stall): one cheap test for the common
        # case (all tensors on this device, contiguous), the general bookkeeping only when it fails
        passthrough: Dict[int, torch.Tensor] = {}
        cuda_tensors = all_tensors
        if not all([t.get_device() == dev for t in all_tensors]):
            passthrough = {i: t for i, t in enumerate(all_tensors) if t.get_device() != dev}
            if any(t.is_cuda for t in passthrough.values()):
                raise ValueError("snapshot: the CUDA tensors must live on one device (the engine's)")
            cuda_tensors = [t for i, t in enumerate(all_tensors) if i not in passthrough]
        # the kernel walks contiguous byte ranges; strided tensors are compacted first (rare)
        if not all([t.is_contiguous() for t in cuda_tensors]):
            cuda_tensors = [t if t.is_contiguous() else t.detach().contiguous() for t in cuda_tensors]
        mask = self._narrow_mask(cuda_tensors, narrow) if narrow else None
        if container is None:
            from .fastsave import zero_copy_enabled

            container = zero_copy_enabled()
        container = bool(container) and not passthrough and len(cuda_tensors) > 0
        if container and self._spare_slots() <= 1:
            # every published checkpoint pins one slot until its file is deleted.  Keep the last slot that is not somebody's
            # checkpoint for copying saves, instead of publishing it too and paying a 16 GB re-pin on the next save
            container = False
        plan = self._plan_for(cuda_tensors, mask, container)

        if trace is not None:
            trace["planned"] = _time.perf_counter()
        stream = self._current_stream()
        staging = self._ensure_staging(plan.staging_bytes)
        tail_room = 0
        if container:
            from .ptzip import slot_tail_room

            tail_room = slot_tail_room(len(cuda_tensors))
        crc = None
        need = plan.staging_bytes
        if gpu_crc_enabled() and not passthrough and len(cuda_tensors) > 0:
            crc = getattr(plan, "_crc", None)
            if crc is None:
                crc = plan._crc = CrcPlan(plan.offsets, plan.packed_nbytes, self.device)
            crc_off = -(-plan.staging_bytes // 64) * 64  # partial values, then the ready word, behind the payload
            ready_off = crc_off + -(-4 * crc.n_values // 8) * 8
            need = ready_off + 8
        slot = self._acquire_slot(need + tail_room)
        if self._staging_free is not None:
            # the previous drain may still be reading staging: order the pack after it on the GPU
            stream_wait_event(stream, self._staging_free)

        start = stop = None
        packed_ev = Event(self.device) if crc is not None else None
        base = slot.drained_total
        if self.timing:
            # separate launches so the pack kernel can be timed on its own (bench / profiling)
            start, stop = Event(self.device, timing=True), Event(self.device, timing=True)
            plan.commit(stream)
            start.record(stream)
            plan.pack(staging.ptr, stream)
            stop.record(stream)
            if packed_ev is not None:
                packed_ev.record(stream)
            self._side.wait_event(stop)
            check(
                self.lib.nvrx_drain(
                    slot.buf.data_ptr, staging.ptr, plan.staging_bytes, self.drain_chunk, slot.buf.progress_ptr, base,
                    self._side.handle, slot.done_event.handle,
                ),
                "nvrx_drain",
            )
        else:
            # pipelined: chunk c is copied out as soon as its sub-launch of the pack kernel has finished
            check(
                self.lib.nvrx_snapshot(
                    plan._h, staging.ptr, slot.buf.data_ptr, self.drain_chunk, slot.buf.progress_ptr, base, stream,
                    self._side.handle, packed_ev.handle if packed_ev is not None else None, slot.done_event.handle,
                ),
                "nvrx_snapshot",
            )
        if trace is not None:
            trace["launched"] = _time.perf_counter()
        self.launches += (plan.last_launches() if not self.timing else 1) if plan.n_tiles else 0
        slot.drained_total = base + plan.staging_bytes
        self._staging_free = slot.done_event
        crc_info = None
        if crc is not None:
            # checksum kernel on a third stream, concurrent with the drain: reads staging once more, sends one 32-bit value per
            # 64 KiB and finally the ready word (= this snapshot's progress target) to the slot
            if self._aux is None:
                self._aux = Stream(self.device)
            self._aux.wait_event(packed_ev)
            crc.run(staging.ptr, slot.buf.data_ptr + crc_off, slot.buf.data_ptr + ready_off, slot.drained_total, self._aux.handle)
            self.launches += 1
            crc_done = Event(self.device)
            crc_done.record(self._aux.handle)
            # staging is free for the next pack only when the drain AND the checksum kernel are through with it
            self._side.wait_event(crc_done)
            free_ev = Event(self.device)
            free_ev.record(self._side.handle)
            self._staging_free = free_ev
            crc_info = {"offset": crc_off, "n_values": crc.n_values, "ready_offset": ready_off, "ready_value": slot.drained_total}

        # the layout only depends on the plan and the shapes: built once per (plan, shapes), not per snapshot
        shapes = [t.shape for t in cuda_tensors]
        dtypes = [t.dtype for t in cuda_tensors]
        cached = plan.__dict__.get("_layout")
        if cached is not None and cached[0] == shapes and cached[2] == dtypes:
            layout = cached[1]
        else:
            layout = PackedLayout(
                shapes=[tuple(sh) for sh in shapes],
                dtypes=[dtype_name(torch.bfloat16 if (mask is not None and nr) else t.dtype)
                        for t, nr in zip(cuda_tensors, mask if mask is not None else [False] * len(cuda_tensors))],
                src_dtypes=[dtype_name(t.dtype) for t in cuda_tensors],
                offsets=list(plan.offsets),
                packed_nbytes=list(plan.packed_nbytes),
                total_bytes=plan.staging_bytes,
                align=self.align,
            )
            plan.__dict__["_layout"] = (shapes, layout, dtypes)
        return Snapshot(
            engine=self, slot=slot, layout=layout, progress_target=slot.drained_total, passthrough=passthrough,
            n_total=len(all_tensors), pack_start=start, pack_stop=stop, crc_info=crc_info,
        )

    # ---- restore --------------------------------------------------------------------------------
    def restore(
        self,
        host_tensors: Sequence[torch.Tensor],
        *,
        widen_to: Optional[Sequence[torch.dtype]] = None,
        out: Optional[Sequence[torch.Tensor]] = None,
        resident: Optional[Tuple[_Slot, Sequence[int]]] = None,
        file_source: Optional[Tuple[str, Sequence[int]]] = None,
        expect_crcs: Optional[Sequence[int]] = None,
    ) -> List[torch.Tensor]:
        """CPU tensors -> CUDA tensors of this device with one H2D copy and one scatter kernel.

        ``widen_to[i] == torch.float32`` for a bf16 host tensor widens it in the scatter kernel (exact).
        ``resident`` (from :meth:`resident_source`): the tensors' bytes already sit in that pinned slot at those payload
        offsets (the checkpoint file is a hard link to the slot), so the gather into a pinned buffer is skipped and the
        H2D reads the slot directly.
        ``file_source = (path, file offsets)`` (from ``ptzip.tensor_offsets_in_file``): fill the pinned slot with parallel
        ``pread`` from the checkpoint file instead of a memcpy from the tensors' mmap (no page-by-page faults).
        ``expect_crcs[i]``: crc32 the bytes of tensor i must have (from the file's directory; 0 = unknown).  The checksum
        kernel sums what actually ARRIVED in HBM, so a flipped bit in the file, the page cache, the pinned slot or on the way
        over PCIe fails the restore (``SnapError``) instead of silently resuming training from corrupt weights."""
        host_tensors = [t.detach() for t in host_tensors]
        target_dtypes = [
            (widen_to[i] if widen_to is not None and widen_to[i] is not None else t.dtype)
            for i, t in enumerate(host_tensors)
        ]
        mask = [td == torch.float32 and t.dtype == torch.bfloat16 and t.numel() > 0 for t, td in zip(host_tensors, target_dtypes)]
        dev = torch.device("cuda", self.device)
        if out is None:
            out = [torch.empty(t.shape, dtype=td, device=dev) for t, td in zip(host_tensors, target_dtypes)]
        else:
            out = list(out)
            for o, t, td in zip(out, host_tensors, target_dtypes):
                assert o.is_cuda and o.is_contiguous() and o.dtype == td and o.shape == t.shape
        if resident is None and file_source is not None and not (expect_crcs is not None and any(expect_crcs)):
            return self._restore_from_file(out, mask, file_source)
        keep_busy = False
        if resident is None and file_source is None:
            # Host tensors that ARE views of one of this engine's pinned slots (a state dict that was just saved: after
            # ``save()`` its tensors are windows into the snapshot slot, and the reference's tests restore exactly such an
            # object, tests/checkpointing/unit/test_basic_local.py:62-64) are restored from where they lie.  Gathering them into
            # "a free slot" could pick the very slot they live in and overwrite them while they are being read.
            held = self._slot_holding(host_tensors)
            if held is not None and held[1] is None:
                host_tensors = [t.clone() for t in host_tensors]  # views of a slot in no usable order: take them out first
            elif held is not None:
                resident, keep_busy = held, held[0].busy
        if resident is not None:
            slot, offsets = resident
            plan = self._plan_for(out, mask, offsets=list(offsets))
            assert plan.staging_bytes <= slot.buf.capacity and (keep_busy or not slot.busy)
            slot.busy = True  # nobody may pick it while the H2D reads it (it is also protected by its link count)
            self.resident_restores += 1
        else:
            plan = self._plan_for(out, mask)
            slot = self._acquire_slot(plan.staging_bytes)
        staging = self._ensure_staging(plan.staging_bytes)
        try:
            if resident is None and file_source is not None:
                path, file_offs = file_source
                live = [(off, nb, fo) for off, nb, fo in zip(plan.offsets, plan.packed_nbytes, file_offs) if nb]
                fd = os.open(path, os.O_RDONLY)
                try:
                    slot.buf.readv_fd([x[0] for x in live], [x[1] for x in live], [x[2] for x in live], fd, threads=self.prefault_threads or 8)
                finally:
                    os.close(fd)
            elif resident is None:
                # gather the CPU tensors into the pinned slot at the plan's offsets (no-op cost when the
                # tensors already are views of one packed buffer with this layout)
                srcs = [t if t.is_contiguous() else t.contiguous() for t in host_tensors]
                base = slot.buf.data_ptr
                todo = [(s.data_ptr(), nb, off) for s, off, nb in zip(srcs, plan.offsets, plan.packed_nbytes) if nb and s.data_ptr() != base + off]
                if todo:
                    slot.buf.gather([x[0] for x in todo], [x[1] for x in todo], [x[2] for x in todo], threads=self.prefault_threads or 8)
            stream = self._current_stream()
            if self._staging_free is not None:
                stream_wait_event(stream, self._staging_free)
            check(
                self.lib.nvrx_fill(staging.ptr, slot.buf.data_ptr, plan.staging_bytes, self.drain_chunk, stream, None),
                "nvrx_fill",
            )
            crc = values = None
            if expect_crcs is not None and any(expect_crcs):
                assert len(expect_crcs) == len(out)
                crc = CrcPlan(plan.offsets, plan.packed_nbytes, self.device)
                values = torch.zeros(crc.n_values + 2, dtype=torch.int32).pin_memory()
                crc.run(staging.ptr, values.data_ptr(), 0, 0, stream)  # same stream: after the H2D, before anything reuses staging
                self.launches += 1
            plan.scatter(staging.ptr, stream)
            self.launches += 1 if plan.n_tiles else 0
            done = Event(self.device)
            done.record(stream)
            self._staging_free = done
            done.synchronize()  # the pinned slot is reused; restore is a blocking call like the reference's
            if crc is not None:
                # the < 512 left-over bytes per tensor are summed from the pinned slot the H2D read from
                got = finish_crcs(plan.offsets, plan.packed_nbytes, values.data_ptr(), crc.n_values, slot.buf.data_ptr)
                crc.close()
                bad = [i for i, (g, e, nb) in enumerate(zip(got, expect_crcs, plan.packed_nbytes)) if nb and e and g != e]
                if bad:
                    raise SnapError(
                        _cabi.E_STATE, "verifying restored tensors",
                        f"crc32 mismatch on {len(bad)} of {len(out)} tensors (first: #{bad[0]}, got {got[bad[0]]:#010x}, "
                        f"file says {expect_crcs[bad[0]]:#010x}) -- the checkpoint is corrupt",
                    )
        finally:
            if not keep_busy:
                self._release(slot)
        return out

    def _slot_holding(self, host_tensors: Sequence[torch.Tensor]):
        """``(slot, payload offsets)`` when every non-empty tensor is a contiguous view into ONE slot of this engine, ascending
        and 16-byte aligned (a plan can read them in place); ``(slot, None)`` when they touch a slot in any other way; None
        when they have nothing to do with the slots."""
        live = [t for t in host_tensors if t.numel()]
        if not live:
            return None
        for slot in self._slots:
            if slot.buf is None:
                continue
            base, cap = slot.buf.data_ptr, slot.buf.capacity
            inside = [base <= t.data_ptr() < base + cap for t in live]
            if not any(inside):
                continue
            if not all(inside):
                return slot, None
            offs, end = [], 0
            for t in host_tensors:
                nb = t.numel() * t.element_size()
                off = (t.data_ptr() - base) if nb else -(-end // 16) * 16
                if nb and (off < end or off % 16 or off + nb > cap or not t.is_contiguous()):
                    return slot, None
                offs.append(off)
                end = off + nb
            return slot, offs
        return None

    RESTORE_CHUNK = int(os.environ.get("NVRX_B200_RESTORE_CHUNK_MB", "64")) << 20
    RESTORE_RING = int(os.environ.get("NVRX_B200_RESTORE_RING", "4"))
    RESTORE_THREADS = int(os.environ.get("NVRX_B200_RESTORE_THREADS", "0"))

    def _restore_from_file(self, out: List[torch.Tensor], mask: Sequence[bool], file_source) -> List[torch.Tensor]:
        """File -> GPU tensors without a snapshot-sized host buffer (``nvrx_fill_from_fd``): a pool of readers fills a small
        ring of pinned chunks from the checkpoint file while the chunks already read travel to the device; one scatter
        kernel at the end.  A freshly restarted process does not have to create and page-lock a 16 GB slot first (~2 s)."""
        import time as _time

        path, file_offs = file_source
        t0 = _time.perf_counter()
        plan = self._plan_for(out, mask)
        t1 = _time.perf_counter()
        staging = self._ensure_staging(plan.staging_bytes)
        t2 = _time.perf_counter()
        live = [(off, nb, fo) for off, nb, fo in zip(plan.offsets, plan.packed_nbytes, file_offs) if nb]
        stream = self._current_stream()
        if self._staging_free is not None:
            stream_wait_event(stream, self._staging_free)
        threads = self.RESTORE_THREADS or max(self.prefault_threads, min(32, os.cpu_count() or 1))
        fd = os.open(path, os.O_RDONLY)
        try:
            check(
                self.lib.nvrx_fill_from_fd(
                    staging.ptr, plan.staging_bytes, fd, len(live), _u64_array([x[0] for x in live]), _u64_array([x[1] for x in live]),
                    _u64_array([x[2] for x in live]), self.RESTORE_CHUNK, self.RESTORE_RING, threads, self.device, stream,
                ),
                "nvrx_fill_from_fd",
            )
        finally:
            os.close(fd)
        t3 = _time.perf_counter()
        plan.scatter(staging.ptr, stream)
        self.launches += 1 if plan.n_tiles else 0
        self.file_restores += 1
        done = Event(self.device)
        done.record(stream)
        self._staging_free = done
        done.synchronize()  # restore is a blocking call like the reference's
        if self.trace is not None:
            self.trace["restore"] = {"plan_s": t1 - t0, "staging_s": t2 - t1, "file_to_device_s": t3 - t2, "scatter_s": _time.perf_counter() - t3}
        return out

    def resident_source(self, path, host_tensors: Sequence[torch.Tensor]) -> Optional[Tuple[_Slot, List[int]]]:
        """``(slot, payload offsets)`` when the checkpoint file ``path`` is a hard link to one of this engine's live,
        pinned slots (zero-copy persistence; e.g. an in-process restart that reloads the checkpoint it wrote itself) and
        ``host_tensors`` are the tensors ``torch.load(path, mmap=True)`` returned, in file order; else None."""
        from .ptzip import SLOT_PREFIX, tensor_offsets_in_file

        for slot in self._slots:
            if slot.buf is None or slot.busy or not slot.buf.name:
                continue
            try:
                if not os.path.samefile("/dev/shm" + slot.buf.name, path):
                    continue
            except OSError:
                continue
            offs = tensor_offsets_in_file(path, host_tensors)
            if offs is None or any(o < SLOT_PREFIX for o in offs):
                return None
            return slot, [o - SLOT_PREFIX for o in offs]
        return None

    def restore_from_staging(self, plan: Plan, staging_ptr: int) -> None:
        """Scatter a staging buffer that is already on the device (replica retrieval path)."""
        plan.scatter(staging_ptr, self._current_stream())
        self.launches += 1 if plan.n_tiles else 0

    def trim(self) -> None:
        """Give memory back between checkpoints: the device staging buffer (as large as the snapshot) and every host slot
        that is not owned by an unfinalized save.  The next snapshot re-creates what it needs (cudaMalloc + memset of the
        staging buffer: milliseconds; pinning a 16 GB slot: ~2 s)."""
        if self._staging is not None:
            if self._staging_free is not None:
                self._staging_free.synchronize()
            self._staging.close()
            self._staging = None
        for s in self._slots:
            if not s.busy and s.buf is not None:
                if s.done_event is not None:
                    s.done_event.synchronize()
                s.__dict__.pop("_exchange_views", None)
                s.buf.close()
                s.buf = None

    def close(self) -> None:
        if os.getpid() != self._pid:
            return
        for plan in self._plans.values():
            if getattr(plan, "_crc", None) is not None:
                plan._crc.close()
            plan.close()
        self._plans.clear()
        for s in self._slots:
            if s.done_event is not None:
                try:
                    s.done_event.synchronize()
                except SnapError:
                    pass
            if s.buf is not None:
                s.buf.close()
                s.buf = None
        if self._staging is not None:
            self._staging.close()
            self._staging = None
        for ptr in [p for pm in getattr(self, "_peer_maps", {}).values() for p in pm["imported"]]:
            self.lib.nvrx_ipc_close(self.device, ptr)
        self._peer_maps = {}
        for attr in ("_exchange_buf", "_p2p_buf", "_ring_buf"):
            buf = getattr(self, attr, None)
            if buf is not None:
                buf.close()
                setattr(self, attr, None)


import atexit  # noqa: E402

atexit.register(SnapshotEngine.shutdown_all)  # unlink the shm slots of a normally exiting trainer


def open_snapshot_views(desc: dict, timeout_ms: int = -1) -> Tuple[HostBuffer, List[torch.Tensor]]:
    """Writer-process side: map the slot by name, wait (CPU only) for the drain, return tensor views."""
    hb = HostBuffer.open(desc["shm_name"])
    hb.wait(desc["progress_target"], timeout_ms)
    layout: PackedLayout = desc["layout"]
    return hb, host_views(layout, hb)
