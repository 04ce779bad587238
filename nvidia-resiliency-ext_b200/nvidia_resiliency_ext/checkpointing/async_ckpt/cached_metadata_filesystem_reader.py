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
See ``SnapshotEngine.load_boxes``."""

import dataclasses
import os
from typing import Dict, Optional, Union

import torch
from torch.distributed.checkpoint import FileSystemReader, Metadata
from torch.distributed.checkpoint.planner import LoadItemType, LoadPlan, LoadPlanner
from torch.futures import Future

# dtypes the engine converts between on the device (any other dtype mismatch takes FileSystemReader's path)
_DEVICE_CAST_DTYPES = (torch.float32, torch.bfloat16, torch.float16)


class CachedMetadataFileSystemReader(FileSystemReader):
    _metadata_cache: Dict[str, Metadata] = {}

    def __init__(self, path: Union[str, os.PathLike], cache_metadata: bool = True, *, load_on_engine: bool = False) -> None:
        """``cache_metadata=False`` makes this a plain ``FileSystemReader`` (every ``read_metadata`` hits the disk).
        ``load_on_engine=True``: tensor items bound for CUDA tensors of the current device, stored without storage
        transforms and with their target's dtype (or fp32 / bf16 / fp16 into another of these three, converted on the
        device), are loaded by the snapshot engine; everything else takes ``FileSystemReader``'s path.  Raises like ``SnapshotEngine`` when there is no CUDA device or no engine library (no silent fallback)."""
        super().__init__(path=path)
        self._cache_key: Optional[str] = os.path.abspath(os.fspath(path)) if cache_metadata else None
        self._load_on_engine = bool(load_on_engine)
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

    def read_data(self, plan: LoadPlan, planner: LoadPlanner) -> Future:
        if not self._load_on_engine:
            return super().read_data(plan, planner)
        from ..b200.engine import BoxLoad, SnapshotEngine
        from ..b200.ptzip import read_tensor_record

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
        if mine:
            entries, chunks, fds = [], {}, {}
            try:
                for req, info, target, saved_dtype in mine:
                    path = os.fspath(self.fs.concat_path(self.path, info.relative_path))
                    chunk = chunks.get((path, info.offset))
                    if chunk is None:
                        if path not in fds:
                            fds[path] = os.open(path, os.O_RDONLY)
                        chunk = chunks[(path, info.offset)] = read_tensor_record(fds[path], info.offset, info.length)
                    if chunk.dtype != saved_dtype:
                        raise ValueError(f"{req.storage_index.fqn}: stored as {chunk.dtype}, metadata says {saved_dtype}")
                    if tuple(target.shape) != tuple(req.lengths):
                        raise AssertionError(f"req {req.storage_index} mismatch sizes {tuple(target.shape)} vs {tuple(req.lengths)}")
                    src_offset = chunk.storage_offset + sum(o * s for o, s in zip(req.storage_offsets, chunk.stride))
                    entries.append(
                        BoxLoad(path, chunk.data_off, chunk.numel * chunk.dtype.itemsize, src_offset, chunk.stride, target,
                                None if chunk.dtype == target.dtype else chunk.dtype)
                    )
            finally:
                for fd in fds.values():
                    os.close(fd)
            engine.load_boxes(entries)  # returns after the device work is done
            for req, _, target, _ in mine:
                planner.commit_tensor(req, target)
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
