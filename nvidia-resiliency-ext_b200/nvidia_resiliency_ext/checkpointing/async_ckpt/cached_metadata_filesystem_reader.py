"""``FileSystemReader`` that reads a checkpoint's ``.metadata`` once per process.

Same role as reference ``checkpointing/async_ckpt/cached_metadata_filesystem_reader.py`` (``CachedMetadataFileSystemReader``
``:24``): several loads of one checkpoint directory (model, optimizer, ... loaded by separate ``dcp.load`` calls) unpickle the
global metadata only the first time.  The cache is per class, keyed by the absolute checkpoint path.

``load_on_engine=True`` (opt-in) loads the tensor items whose targets are CUDA tensors of this device through the H100
snapshot engine instead of ``FileSystemReader.read_data``'s per-item ``torch.load`` + ``narrow`` + pageable ``copy_``: only
the byte span each read item needs goes file -> pinned ring -> HBM, and one box-scatter kernel per staging batch writes
every (possibly resharded, possibly non-contiguous) target view.  Items saved as fp32, bf16 or fp16 and loaded into a
target of another of the three dtypes (an fp32 checkpoint into a bf16 model, bf16 weights into fp32 master parameters) are
converted by that kernel, rounding to nearest even like ``Tensor.to``; bits match the stock reader except for NaN payloads.
See ``SnapshotEngine.load_boxes``.

``verify=True`` checks every tensor item the load reads against the CRC-32 its storage record carries in the ``.distcp``
file's ZIP directory (``torch.save`` fills it in; ``torch.load`` never checks it), so a bit flipped on disk, in the page
cache, in host memory or on PCIe raises ``SnapError`` ("crc32 mismatch ...") instead of becoming a weight.  Items loaded
by the engine are summed on the GPU over the bytes that reached HBM; the other tensor items are read a second time and
summed on the host before ``FileSystemReader.read_data`` runs.  Each archive's ``data.pkl`` (the storage offset, size and
stride that decide where the bytes go) is checked against its own CRC-32 field whenever the engine parses it.  BYTE_IO
items, items with storage transforms and items whose records were written without checksums cannot be checked: they
are counted, as items, and reported with one warning per ``read_data``."""

import dataclasses
import os
import warnings
import zlib
from typing import Dict, Optional, Union

import torch
from torch.distributed.checkpoint import FileSystemReader, Metadata
from torch.distributed.checkpoint.planner import LoadItemType, LoadPlan, LoadPlanner
from torch.futures import Future

# dtypes the engine converts between on the device (any other dtype mismatch takes FileSystemReader's path)
_DEVICE_CAST_DTYPES = (torch.float32, torch.bfloat16, torch.float16)


class CachedMetadataFileSystemReader(FileSystemReader):
    _metadata_cache: Dict[str, Metadata] = {}

    def __init__(self, path: Union[str, os.PathLike], cache_metadata: bool = True, *, load_on_engine: bool = False,
                 verify: bool = False) -> None:
        """``cache_metadata=False`` makes this a plain ``FileSystemReader`` (every ``read_metadata`` hits the disk).
        ``load_on_engine=True``: tensor items bound for CUDA tensors of the current device, stored without storage
        transforms and with their target's dtype (or fp32 / bf16 / fp16 into another of these three, converted on the
        device), are loaded by the snapshot engine; everything else takes ``FileSystemReader``'s path.  Raises like ``SnapshotEngine`` when there is no CUDA device or no engine library (no silent fallback).
        ``verify=True``: check every tensor item read against its record's CRC-32 (module docstring); a mismatch raises
        ``SnapError`` before any item of the ``read_data`` call is committed to the planner.  ``last_verify`` then holds
        the records checked on the GPU and on the host and the items left unverified."""
        super().__init__(path=path)
        self._cache_key: Optional[str] = os.path.abspath(os.fspath(path)) if cache_metadata else None
        self._load_on_engine = bool(load_on_engine)
        self._verify = bool(verify)
        self.last_verify: Optional[dict] = None
        self._loaded_metadata: Optional[Metadata] = None
        if self._load_on_engine:
            from ..b200 import _cabi

            _cabi.lib()
            if not torch.cuda.is_available():
                raise _cabi.SnapError(_cabi.E_STATE, "load_on_engine", "no CUDA device - the engine load path has no CPU fallback")

    def read_metadata(self) -> Metadata:
        key = self._cache_key
        if key is None:
            return super().read_metadata()
        cache = type(self)._metadata_cache
        if key not in cache:
            cache[key] = super().read_metadata()
        return cache[key]

    def set_up_storage_reader(self, metadata: Metadata, is_coordinator: bool, *args, **kwargs) -> None:
        super().set_up_storage_reader(metadata, is_coordinator, *args, **kwargs)
        self._loaded_metadata = metadata

    def _read_record(self, fd: int, path: str, offset: int, length: int, names):
        """``read_tensor_record``; with ``verify=True`` a ``data.pkl`` that does not match its CRC-32 field (it says where
        the item's bytes go) is reported as the items' crc32 mismatch."""
        from ..b200._cabi import E_STATE, SnapError
        from ..b200.ptzip import RecordChecksumError, read_tensor_record

        try:
            return read_tensor_record(fd, offset, length)
        except RecordChecksumError as e:
            if not self._verify:
                raise
            raise SnapError(
                E_STATE, "verifying loaded items",
                f"crc32 mismatch on {', '.join(names)} in {path} at {e.member} (header offset {e.header_off}): got "
                f"{e.got:#010x}, file says {e.expected:#010x} -- the checkpoint is corrupt",
            ) from e

    def _verify_on_host(self, items, stats: dict) -> None:
        """Read each tensor record of ``items`` (once per record) and compare its zlib CRC-32 with the directory's field;
        BYTE_IO items, items with storage transforms and items of records written without checksums count as
        unverified."""
        from ..b200._cabi import E_STATE, SnapError

        records: Dict[tuple, list] = {}
        for req in items:
            info = self.storage_data[req.storage_index]
            if req.type != LoadItemType.TENSOR or getattr(info, "transform_descriptors", None):
                stats["unverified"] += 1
                continue
            path = os.fspath(self.fs.concat_path(self.path, info.relative_path))
            records.setdefault((path, info.offset, info.length), []).append(req.storage_index.fqn)
        for (path, offset, length), names in records.items():
            fd = os.open(path, os.O_RDONLY)
            try:
                rec = self._read_record(fd, path, offset, length, names)
                if rec.record_len and rec.crc32 == 0:
                    stats["unverified"] += len(names)  # written without checksums
                    continue
                crc, pos, end = 0, rec.data_off, rec.data_off + rec.record_len
                while pos < end:
                    data = os.pread(fd, min(64 << 20, end - pos), pos)
                    if not data:
                        break
                    crc = zlib.crc32(data, crc)
                    pos += len(data)
            finally:
                os.close(fd)
            if crc != rec.crc32:
                raise SnapError(
                    E_STATE, "verifying loaded items",
                    f"crc32 mismatch on {', '.join(names)} in {path} at record offset {rec.data_off}: got {crc:#010x}, "
                    f"file says {rec.crc32:#010x} -- the checkpoint is corrupt",
                )
            stats["host_records"] += 1

    def _report_unverified(self, stats: dict) -> None:
        self.last_verify = stats
        if stats["unverified"]:
            warnings.warn(
                f"{stats['unverified']} checkpoint items were loaded without a checksum check (BYTE_IO items, items with "
                "storage transforms or items whose records were written without CRC-32)",
                stacklevel=3,
            )

    def read_data(self, plan: LoadPlan, planner: LoadPlanner) -> Future:
        stats = {"gpu_records": 0, "host_records": 0, "unverified": 0}
        if not self._load_on_engine:
            if self._verify:
                self._verify_on_host(plan.items, stats)
                self._report_unverified(stats)
            return super().read_data(plan, planner)
        from ..b200.engine import BoxLoad, SnapshotEngine

        engine = SnapshotEngine.get()
        saved_md = self._loaded_metadata.state_dict_metadata if self._loaded_metadata is not None else {}
        mine, rest = [], []
        for req in plan.items:
            info = self.storage_data[req.storage_index]
            saved = saved_md.get(req.storage_index.fqn)
            if req.type == LoadItemType.TENSOR and not getattr(info, "transform_descriptors", None) and saved is not None:
                target = planner.resolve_tensor(req).detach()
                saved_dtype = saved.properties.dtype
                same = target.dtype == saved_dtype
                cast = target.dtype in _DEVICE_CAST_DTYPES and saved_dtype in _DEVICE_CAST_DTYPES
                if target.is_cuda and target.get_device() == engine.device and (same or cast):
                    mine.append((req, info, target, saved_dtype))
                    continue
            rest.append(req)
        if self._verify:  # the stock-path items first: every check is done before anything is committed
            self._verify_on_host(rest, stats)
        if mine:
            entries, chunks, fds = [], {}, {}
            try:
                for req, info, target, saved_dtype in mine:
                    path = os.fspath(self.fs.concat_path(self.path, info.relative_path))
                    chunk = chunks.get((path, info.offset))
                    if chunk is None:
                        if path not in fds:
                            fds[path] = os.open(path, os.O_RDONLY)
                        chunk = chunks[(path, info.offset)] = self._read_record(
                            fds[path], path, info.offset, info.length, [req.storage_index.fqn])
                    if chunk.dtype != saved_dtype:
                        raise ValueError(f"{req.storage_index.fqn}: stored as {chunk.dtype}, metadata says {saved_dtype}")
                    if tuple(target.shape) != tuple(req.lengths):
                        raise AssertionError(f"req {req.storage_index} mismatch sizes {tuple(target.shape)} vs {tuple(req.lengths)}")
                    if chunk.record_len and chunk.crc32 == 0 and target.numel():
                        stats["unverified"] += 1  # an item of a record written without checksums
                    src_offset = chunk.storage_offset + sum(o * s for o, s in zip(req.storage_offsets, chunk.stride))
                    entries.append(
                        BoxLoad(path, chunk.data_off, chunk.numel * chunk.dtype.itemsize, src_offset, chunk.stride, target,
                                None if chunk.dtype == target.dtype else chunk.dtype,
                                record_crc=chunk.crc32 if self._verify else None, record_len=chunk.record_len,
                                name=req.storage_index.fqn)
                    )
            finally:
                for fd in fds.values():
                    os.close(fd)
            if self._verify:
                engine.load_boxes(entries, verify=True)  # raises on a mismatch, before anything is committed
                stats["gpu_records"] += engine.last_box_load["verified_records"]
            else:
                engine.load_boxes(entries)  # returns after the device work is done
            for req, _, target, _ in mine:
                planner.commit_tensor(req, target)
        if self._verify:
            self._report_unverified(stats)
        if rest:
            return super().read_data(dataclasses.replace(plan, items=rest), planner)
        fut: Future = Future()
        fut.set_result(None)
        return fut

    @classmethod
    def clear_metadata_cache(cls, path: Union[str, os.PathLike, None] = None) -> None:
        """Forget one checkpoint directory (e.g. after it was overwritten), or everything when ``path`` is None."""
        if path is None:
            cls._metadata_cache.clear()
        else:
            cls._metadata_cache.pop(os.path.abspath(os.fspath(path)), None)
