"""``torch.save`` files -> the GPU through the snapshot engine (``TorchAsyncCheckpoint.load``).

``torch.load(f, map_location="cuda")`` unpickles, reads every record on one thread into pageable memory and then copies each
tensor to the device on its own; ``load_state_dict`` copies each once more.  Here the archive is planned without reading
any payload -- ``torch.load(mmap=True)`` (weights_only: no code runs) gives every tensor's storage, element offset, sizes,
strides and dtype, the file mapping's base turns each storage into its record's file offset, and the ZIP directory gives the
record's length and CRC-32 field -- and the bytes then travel on the engine's existing paths:

* new tensors: one CUDA storage per file record, filled by ``SnapshotEngine.restore`` (parallel ``pread`` -> pinned ring ->
  HBM -> one scatter, or the checksum path with ``verify``; a file that is a hard link to one of this process's pinned
  slots is read in place), then the views are built on those storages with ``set_``;
* in place: one ``BoxLoad`` per tensor into the live targets (any strides, fp32 / bf16 / fp16 converted on the device),
  ``SnapshotEngine.load_boxes``.

The planning half (:func:`plan_archive`, :func:`match_keys`, :func:`on_engine`) runs without CUDA."""

from __future__ import annotations

import copy
import os
import time
import warnings
import zlib
from dataclasses import dataclass, field
from typing import Any, Dict, List, NamedTuple, Optional, Tuple

import torch

from . import ptzip
from .engine import BOX_CASTS

BOX_MAXDIM = 8  # NVRX_BOX_MAXDIM (include/nvrx_snap.h): targets with more dims are copied with ``Tensor.copy_``


@dataclass
class StorageRecord:
    """One ``data/<key>`` record of the archive: where its bytes lie in the file and what its directory entry says."""

    key: int
    file_off: int
    nbytes: int
    crc32: int  # CRC-32 field in the central directory (0 on a non-empty record: written without one)
    record_len: int


@dataclass
class TensorEntry:
    """A tensor of the loaded object, at nested ``path``, as a view of ``storages[storage]``."""

    path: Tuple[Any, ...]
    storage: int
    storage_offset: int  # elements
    size: Tuple[int, ...]
    stride: Tuple[int, ...]
    dtype: torch.dtype


@dataclass
class ArchivePlan:
    path: str
    obj: Any  # what torch.load(mmap=True) returned: CPU tensors on the file's mapping
    storages: List[StorageRecord] = field(default_factory=list)
    host_storages: List[torch.UntypedStorage] = field(default_factory=list)  # parallel to ``storages``
    entries: List[TensorEntry] = field(default_factory=list)
    host_tensors: List[torch.Tensor] = field(default_factory=list)  # parallel to ``entries``
    plan_ms: float = 0.0  # host time of plan_archive when timed by load()


class IncompatibleKeys(NamedTuple):
    missing_keys: List[str]
    unexpected_keys: List[str]


def key_name(path: Tuple[Any, ...]) -> str:
    """``("model", "layers", 0, "w")`` -> ``"model.layers.0.w"``."""
    return ".".join(str(p) for p in path)


def tensor_leaves(obj) -> List[Tuple[Tuple[Any, ...], torch.Tensor]]:
    """``(path, tensor)`` of every tensor reachable through dicts, lists and tuples, depth first."""
    out: List[Tuple[Tuple[Any, ...], torch.Tensor]] = []
    on_stack = set()

    def walk(x, path):
        if isinstance(x, torch.Tensor):
            out.append((path, x))
        elif isinstance(x, (dict, list, tuple)) and id(x) not in on_stack:
            on_stack.add(id(x))
            for k, v in (x.items() if isinstance(x, dict) else enumerate(x)):
                walk(v, path + (k,))
            on_stack.discard(id(x))

    walk(obj, ())
    return out


def replace_tensors(obj, new: Dict[int, torch.Tensor]):
    """A copy of ``obj`` whose tensors are ``new[id(tensor)]``; containers keep their types, other leaves are shared."""
    memo: Dict[int, Any] = {}

    def rebuild(x):
        if isinstance(x, torch.Tensor):
            return new[id(x)]
        if id(x) in memo:
            return memo[id(x)]
        if isinstance(x, (dict, list)):
            out = memo[id(x)] = copy.copy(x)  # OrderedDict and other subclasses keep their type
            for k, v in (x.items() if isinstance(x, dict) else enumerate(x)):
                out[k] = rebuild(v)
            return out
        if isinstance(x, tuple):
            items = [rebuild(v) for v in x]
            out = memo[id(x)] = type(x)(*items) if hasattr(x, "_fields") else type(x)(items)
            return out
        return x

    return rebuild(obj)


def _file_path(f) -> str:
    if isinstance(f, (str, os.PathLike)):
        return os.fspath(f)
    name = getattr(f, "name", None)
    if isinstance(name, str) and os.path.isfile(name):
        return name
    raise ValueError("the engine load reads the checkpoint by file offsets: pass a path (or a file object opened on one)")


def plan_archive(f) -> ArchivePlan:
    """Plan the load of a ``torch.save`` file without reading its payload (CPU only).  Raises ``ValueError`` when a storage
    cannot be placed in the file or a tensor is held by something other than dicts, lists and tuples."""
    path = _file_path(f)
    seen: List[torch.UntypedStorage] = []

    def keep(storage, location):  # every storage once, in the order the unpickler meets them; stays on the mapping
        seen.append(storage)
        return storage

    obj = torch.load(path, mmap=True, map_location=keep, weights_only=True)
    plan = ArchivePlan(path=path, obj=obj)
    if seen:
        base = ptzip._mapping_base(path, seen[0].data_ptr())
        if base is None:
            raise ValueError(f"{path}: the file's mapping was not found in this process")
        reader = torch._C.PyTorchFileReader(path)
        by_off = {reader.get_record_offset(n): int(n[5:]) for n in reader.get_all_records() if n.startswith("data/")}
        del reader
        import zipfile

        with zipfile.ZipFile(path) as zf:
            infos = ptzip._data_records(zf)
        for st in seen:
            off = st.data_ptr() - base
            key = by_off.get(off)
            if key is None or key not in infos or infos[key].compress_type != zipfile.ZIP_STORED:
                raise ValueError(f"{path}: a storage at file offset {off} is not a stored data record")
            info = infos[key]
            if info.file_size < st.nbytes():
                raise ValueError(f"{path}: record data/{key} is shorter than its storage")
            plan.storages.append(StorageRecord(key, off, st.nbytes(), int(info.CRC), int(info.file_size)))
            plan.host_storages.append(st)
    index = {s.data_ptr(): i for i, s in enumerate(plan.host_storages)}
    for p, t in tensor_leaves(obj):
        i = index[t.untyped_storage().data_ptr()]
        plan.entries.append(TensorEntry(p, i, t.storage_offset(), tuple(t.shape), tuple(t.stride()), t.dtype))
        plan.host_tensors.append(t)
    if len({e.storage for e in plan.entries}) != len(plan.storages) or _reachable_tensors(obj) != {id(t) for t in plan.host_tensors}:
        raise ValueError(f"{path}: some tensors are held by containers other than dicts, lists and tuples")
    return plan


def _reachable_tensors(obj) -> set:
    """``id``s of every tensor reachable from ``obj`` through any object (sets, objects' attributes, ...), not only the
    dicts, lists and tuples :func:`tensor_leaves` walks; classes, modules and functions are not entered."""
    import gc
    import types

    found, seen, stack = set(), set(), [obj]
    while stack:
        x = stack.pop()
        if id(x) in seen:
            continue
        seen.add(id(x))
        if isinstance(x, torch.Tensor):
            found.add(id(x))
        elif not isinstance(x, (type, types.ModuleType, types.FunctionType, types.BuiltinFunctionType)):
            stack.extend(gc.get_referents(x))
    return found


def match_keys(plan: ArchivePlan, into) -> Tuple[List[Tuple[int, torch.Tensor]], List[str], List[str], List[str]]:
    """``(pairs, missing, unexpected, shape mismatches)``: ``pairs`` = (entry index, target) for every saved tensor whose
    nested path holds a tensor in ``into``; ``missing`` = target paths the file lacks; ``unexpected`` = saved paths ``into``
    lacks; mismatches describe pairs whose shapes differ."""
    targets = dict(tensor_leaves(into))
    saved = {e.path: i for i, e in enumerate(plan.entries)}
    pairs, bad = [], []
    for p, i in saved.items():
        t = targets.get(p)
        if t is None:
            continue
        if tuple(t.shape) != plan.entries[i].size:
            bad.append(f"size mismatch for {key_name(p)}: the file has {list(plan.entries[i].size)}, the target {list(t.shape)}")
        pairs.append((i, t))
    missing = [key_name(p) for p in targets if p not in saved]
    unexpected = [key_name(p) for p in saved if p not in targets]
    return pairs, missing, unexpected, bad


def on_engine(target_device: torch.device, target_dtype: torch.dtype, target_dim: int, saved_dtype: torch.dtype,
              engine_device: int) -> bool:
    """True when the engine writes this target (a CUDA tensor of its device with at most ``BOX_MAXDIM`` dims, the saved
    dtype or fp32 / bf16 / fp16 into another of the three); False = ``target.copy_(saved)``."""
    if target_device.type != "cuda" or target_device.index != engine_device or target_dim > BOX_MAXDIM:
        return False
    return target_dtype == saved_dtype or (saved_dtype, target_dtype) in BOX_CASTS


def cuda_device(map_location) -> Optional[torch.device]:
    """The CUDA device ``map_location`` names (``"cuda"``, ``"cuda:k"``, ``torch.device``; the index stays None for the
    current device), or None when it names none (None, the CPU, a dict or a callable: those loads are plain
    ``torch.load``).  Touches no CUDA API."""
    if isinstance(map_location, str):
        map_location = torch.device(map_location)
    if not isinstance(map_location, torch.device) or map_location.type != "cuda":
        return None
    return map_location


def _engine_for(device: Optional[int]):
    """The engine of CUDA device ``device`` (None: the current one); ``SnapError`` without the library or CUDA."""
    from . import _cabi
    from .engine import SnapshotEngine

    _cabi.lib()
    if not torch.cuda.is_available():
        raise _cabi.SnapError(_cabi.E_STATE, "torch load on the engine", "no CUDA device - the engine load path has no CPU fallback")
    return SnapshotEngine.get(device)


def _flat(storage: torch.UntypedStorage) -> torch.Tensor:
    return torch.empty(0, dtype=torch.uint8, device=storage.device).set_(storage)


def _labels(plan: ArchivePlan) -> List[str]:
    """Per storage: the keys of its tensors, the file and the record offset (what a checksum error names)."""
    keys: Dict[int, List[str]] = {}
    for e in plan.entries:
        keys.setdefault(e.storage, []).append(key_name(e.path) or "<root>")
    return [f"{', '.join(keys.get(i, ['?'])[:4])} in {plan.path} at record offset {s.file_off}" for i, s in enumerate(plan.storages)]


def _crc_mismatch(label: str, got: int, want: int):
    from . import _cabi

    return _cabi.SnapError(_cabi.E_STATE, "verifying loaded tensors",
                           f"crc32 mismatch on {label}: got {got:#010x}, file says {want:#010x} -- the checkpoint is corrupt")


def _warn_unverified(n: int) -> None:
    if n:
        warnings.warn(f"{n} checkpoint records were loaded without a checksum check (written without CRC-32)", stacklevel=5)  # the caller of TorchAsyncCheckpoint.load


def load(f, map_location=None, *, into=None, strict: bool = True, verify: bool = False):
    """``TorchAsyncCheckpoint.load``: see there."""
    device = cuda_device(map_location)
    if into is None and device is None:
        return torch.load(f, map_location=map_location)
    if into is not None and map_location is not None:
        raise ValueError("load(into=...) writes into the targets where they are: leave map_location None")
    t0 = time.perf_counter()
    if into is not None:
        cuda = [t for _, t in tensor_leaves(into) if t.is_cuda]
        engine = _engine_for(cuda[0].get_device() if cuda else None)
        return _load_into(_timed_plan(f), engine, into, strict, verify, t0)
    engine = _engine_for(device.index)
    return _load_new(_timed_plan(f), engine, verify, t0)


def _timed_plan(f) -> ArchivePlan:
    t0 = time.perf_counter()
    plan = plan_archive(f)
    plan.plan_ms = (time.perf_counter() - t0) * 1e3
    return plan


def _load_new(plan: ArchivePlan, engine, verify: bool, t0: float):
    dev = torch.device("cuda", engine.device)
    order = sorted(range(len(plan.storages)), key=lambda i: plan.storages[i].file_off)
    out: List[Optional[torch.Tensor]] = [None] * len(plan.storages)
    for i in order:
        out[i] = torch.empty(plan.storages[i].nbytes, dtype=torch.uint8, device=dev)
    host = [_flat(plan.host_storages[i]) for i in order]
    dst = [out[i] for i in order]
    launches, resident_before = engine.launches, engine.resident_restores
    t_host = time.perf_counter() - t0
    stats = {"mode": "new", "plan_ms": plan.plan_ms, "records": len(plan.storages), "entries": len(plan.entries), "fallbacks": 0, "bytes_read": 0,
             "resident": False, "verified_records": 0, "unverified_records": 0}
    total = sum(s.nbytes for s in plan.storages)
    if total:
        expect = names = None
        if verify:
            expect = [plan.storages[i].crc32 if plan.storages[i].nbytes else 0 for i in order]
            stats["verified_records"] = sum(1 for c in expect if c)
            stats["unverified_records"] = sum(1 for i in order if plan.storages[i].nbytes and not plan.storages[i].crc32)
            labels = _labels(plan)
            names = [labels[i] for i in order]
        resident = engine.resident_source(plan.path, host)
        file_source = None if resident is not None else (plan.path, [plan.storages[i].file_off for i in order])
        engine.restore(host, out=dst, resident=resident, file_source=file_source, expect_crcs=expect, crc_names=names)
        stats["resident"] = engine.resident_restores > resident_before
        stats["bytes_read"] = 0 if stats["resident"] else total
    t1 = time.perf_counter()
    views: Dict[int, torch.Tensor] = {}
    for e, t in zip(plan.entries, plan.host_tensors):
        if id(t) in views:
            continue
        v = torch.empty(0, dtype=e.dtype, device=dev).set_(out[e.storage].untyped_storage(), e.storage_offset, e.size, e.stride)
        if isinstance(t, torch.nn.Parameter):
            v = torch.nn.Parameter(v, requires_grad=t.requires_grad)
        elif t.requires_grad:
            v.requires_grad_(True)
        views[id(t)] = v
    result = replace_tensors(plan.obj, views)
    t_host += time.perf_counter() - t1
    stats.update(launches=engine.launches - launches, host_ms=t_host * 1e3, wall_ms=(time.perf_counter() - t0) * 1e3)
    engine.last_torch_load = stats
    _warn_unverified(stats["unverified_records"])
    return result


def _load_into(plan: ArchivePlan, engine, into, strict: bool, verify: bool, t0: float) -> IncompatibleKeys:
    from .engine import BoxLoad, box_span

    pairs, missing, unexpected, bad = match_keys(plan, into)
    if bad or (strict and (missing or unexpected)):
        msgs = list(bad)
        if strict and unexpected:
            msgs.append("unexpected keys: " + ", ".join(unexpected))
        if strict and missing:
            msgs.append("missing keys: " + ", ".join(missing))
        raise RuntimeError(f"error(s) loading {plan.path} into the state dict:\n\t" + "\n\t".join(msgs))
    labels = _labels(plan) if verify else None
    boxes, fallbacks = [], []
    for i, target in pairs:
        e = plan.entries[i]
        if not on_engine(target.device, target.dtype, target.dim(), e.dtype, engine.device):
            fallbacks.append((i, target))
            continue
        st = plan.storages[e.storage]
        boxes.append(BoxLoad(plan.path, st.file_off, st.nbytes, e.storage_offset, e.stride, target.detach(),
                             None if e.dtype == target.dtype else e.dtype, record_crc=st.crc32 if verify else None,
                             record_len=st.record_len, name=key_name(e.path)))
    stats = {"mode": "into", "plan_ms": plan.plan_ms, "records": len({plan.entries[i].storage for i, _ in pairs}), "entries": len(pairs),
             "fallbacks": len(fallbacks), "resident": False, "verified_records": 0, "unverified_records": 0, "host_records": 0}
    if verify:
        # the records the copy_ path reads are checked on the host, before anything is written
        checked = set()
        for i, _ in fallbacks:
            s = plan.entries[i].storage
            st = plan.storages[s]
            if s in checked or not st.nbytes:
                continue
            checked.add(s)
            if not st.crc32:
                stats["unverified_records"] += 1
                continue
            got = zlib.crc32(_flat(plan.host_storages[s]).numpy()) & 0xFFFFFFFF
            if got != st.crc32:
                raise _crc_mismatch(labels[s], got, st.crc32)
            stats["host_records"] += 1
    launches = engine.launches
    t_host = time.perf_counter() - t0
    engine.load_boxes(boxes, verify=verify)
    box = engine.last_box_load or {}
    if verify:
        stats["verified_records"] = box.get("verified_records", 0)
        stats["unverified_records"] += box.get("unverified_records", 0)
    t1 = time.perf_counter()
    with torch.no_grad():
        for i, target in fallbacks:
            target.copy_(plan.host_tensors[i])
    t_host += time.perf_counter() - t1
    # the engine reads each box's span of its record (plus, when verifying, the rest of the records it checks)
    read = sum(box_span(b.target.shape, b.src_strides, (b.src_dtype or b.target.dtype).itemsize) for b in boxes)
    stats.update(bytes_read=read + box.get("verify_extra_bytes", 0) if boxes else 0, batches=box.get("batches", 0) if boxes else 0,
                 launches=engine.launches - launches, host_ms=t_host * 1e3, wall_ms=(time.perf_counter() - t0) * 1e3)
    engine.last_torch_load = stats
    _warn_unverified(stats["unverified_records"])
    return IncompatibleKeys(missing, unexpected)
