"""``TorchAsyncCheckpoint``: ``torch.save`` that returns to training immediately.

API mirror of reference ``checkpointing/async_ckpt/torch_ckpt.py:32-96``.  The reference's ``async_save`` is
per-tensor pinned D2H (``utils.preload_tensors``) + ``torch.cuda.synchronize()`` (``:50``, the training-step
stall) + a request that ships every CPU tensor to the writer.  Here ``async_save`` enqueues one pack kernel
and one side-stream drain, and the request carries only a snapshot descriptor; the writer process waits for
the drain on the shared progress word and then runs ``torch.save`` on views of the pinned slot.
"""

import itertools
import logging

import torch

from ..b200.persist import SnapshotRef, save_snapshot_with_torch
from ..utils import _collect_tensors, _walk_tensors, dict_list_map_outplace, preload_tensors, wrap_for_async
from .core import AsyncCallsQueue, AsyncRequest

logger = logging.getLogger(__name__)


class TorchAsyncCheckpoint(object):
    async_fn = None

    def __init__(self, persistent_queue=True, *, narrow_fp32_to_bf16: bool = False, device_staging: bool = True,
                 check_fence: bool = False):
        """``narrow_fp32_to_bf16`` (new, opt-in): store fp32 tensors as bf16 (halves drain + file size).

        ``device_staging=False`` (new, opt-in): staging-free saves.  ``async_save`` records an event on the current stream
        and hands the copies from the live tensors to the pinned slot to the copy engines on a side stream (plus one small
        kernel for the narrowed and small tensors); no device buffer as large as the state is allocated, and the training
        stream carries nothing but the event record.  The contract: between ``async_save`` and :meth:`fence`, no kernel on
        any stream may write a saved tensor (reads are fine; a training step only writes its parameters and optimizer
        state in the optimizer step, so :meth:`fence_before` ``(optimizer)`` is the usual way to keep it).  The saved
        tensors, and the contiguous temporaries made of non-contiguous ones, are referenced until the save is finalized.

        ``check_fence=True`` (with ``device_staging=False``): detect a broken contract.  :meth:`fence` checksums every
        bit-copied saved tensor on the fenced stream, and finalizing the save compares those CRC-32s with the records of the
        written file; a mismatch raises ``SnapError`` naming the keys and the file.  Narrowed and non-contiguous tensors
        are counted as unchecked (``last_fence_check``).  Needs the writer's record checksums (``NVRX_B200_ZIP_CRC`` not
        0)."""
        from ..b200.engine import gpu_crc_enabled
        from ..b200.persist import zip_crc_enabled

        if not device_staging and gpu_crc_enabled():
            raise ValueError("device_staging=False: NVRX_B200_GPU_CRC=1 checksums the device staging buffer, which this mode "
                             "does not have")
        if check_fence and (device_staging or not zip_crc_enabled()):
            raise ValueError("check_fence=True needs device_staging=False and the writer's record checksums "
                             "(NVRX_B200_ZIP_CRC not 0)")
        self.save = torch.save
        self._async_calls_queue = AsyncCallsQueue(persistent=persistent_queue)
        self._narrow = narrow_fp32_to_bf16
        self._direct = not device_staging
        self._check_fence = check_fence
        self._pending = {}  # call_idx -> Snapshot (host slot released on finalize)
        self._unfenced = []  # staging-free snapshots whose copies may still read the live tensors
        self._checks = {}  # call_idx -> _FenceCheck (check_fence)
        self.last_fence_check = None  # {"path", "checked", "unchecked"} of the last save finalized with check_fence
        # kept for API compatibility: the function the reference would have run in the writer
        TorchAsyncCheckpoint.async_fn = torch.save if persistent_queue else wrap_for_async(torch.save)

    def async_save(self, state_dict, *args, **kwargs):
        """Same calling convention as ``torch.save(state_dict, f, ...)``; returns once the snapshot is
        *enqueued* on the GPU (pack kernel on the current stream, drain on a side stream)."""
        self._reap()
        # a lazy walk: the engine checks each tensor as it comes and launches the pack of a staging range as soon as all of
        # its tensors passed, so walking and checking the rest of the state runs beside the GPU's work
        cuda = (t for t in _walk_tensors(state_dict) if t.is_cuda)
        first = next(cuda, None)
        if first is None:
            # nothing on the GPU (reference config C1): the host tensors go to the writer as they are
            request = AsyncRequest(TorchAsyncCheckpoint.async_fn, (preload_tensors(state_dict), *args), [], kwargs or {})
            self._async_calls_queue.schedule_async_request(request)
            return
        from ..b200.engine import SnapshotEngine

        if self._direct:
            return self._async_save_direct(state_dict, first, cuda, args, kwargs)
        # GPU work first (pack sub-launches + drain are enqueued here), Python bookkeeping while it runs.  Host tensors in the
        # same dict (e.g. ``torch.get_rng_state()``) travel to the writer as they are, like in the reference, whose
        # ``preload_tensors`` maps them through ``.to("cpu")`` = identity (``utils.py:93-94``).
        # (the engine checks that all of them live on ONE device and raises ValueError otherwise)
        snap = SnapshotEngine.get(first.get_device()).snapshot(itertools.chain((first,), cuda), narrow=self._narrow)
        counter = iter(range(snap.n_total))

        def leaf(v):
            if isinstance(v, torch.Tensor):
                return SnapshotRef(next(counter)) if v.is_cuda else v.detach()
            return v

        skeleton = dict_list_map_outplace(leaf, state_dict)
        path, rest = args[0], args[1:]
        request = AsyncRequest(save_snapshot_with_torch, (skeleton, path, snap.descriptor(), *rest), [], kwargs or {})
        idx = self._async_calls_queue.schedule_async_request(request)
        self._pending[idx] = snap

    def _async_save_direct(self, state_dict, first, cuda, args, kwargs):
        """Staging-free ``async_save``: the walk is checked and handed to the engine in one native call
        (``SnapshotEngine.snapshot(direct=True)``); nothing blocks on the GPU."""
        from ..b200.engine import SnapshotEngine

        tensors = [first, *cuda]
        engine = SnapshotEngine.get(first.get_device())
        snap = engine.snapshot(tensors, narrow=self._narrow, direct=True)
        counter = iter(range(snap.n_total))

        def leaf(v):
            if isinstance(v, torch.Tensor):
                return SnapshotRef(next(counter)) if v.is_cuda else v.detach()
            return v

        skeleton = dict_list_map_outplace(leaf, state_dict)
        path, rest = args[0], args[1:]
        request = AsyncRequest(save_snapshot_with_torch, (skeleton, path, snap.descriptor(), *rest), [], kwargs or {})
        idx = self._async_calls_queue.schedule_async_request(request)
        self._pending[idx] = snap
        self._unfenced.append(snap)
        if self._check_fence:
            self._checks[idx] = _FenceCheck(path, _cuda_names(state_dict), tensors, snap)

    def fence(self, stream=None) -> None:
        """Make ``stream`` (default: the current stream) wait on the GPU until every staging-free snapshot taken so far has
        finished reading its tensors.  The host never blocks.  A no-op with device staging or when nothing is pending.
        With ``check_fence``, the first fence after a save also checksums that save's tensors on ``stream``."""
        if not getattr(self, "_unfenced", None):  # (also on an object built without __init__)
            return
        from ..b200.engine import stream_wait_event

        if stream is None:
            stream = torch.cuda.current_stream(self._unfenced[-1].engine.device)
        for check in self._checks.values():
            if check.crcs is None:
                check.run(stream)
        # the copies of all snapshots run in order on one side stream: the last one's read-done event covers the others
        last = self._unfenced[-1].read_done
        stream_wait_event(stream.cuda_stream, last)
        self._unfenced = [s for s in self._unfenced if not s.released and not s.read_done.query()]

    def fence_before(self, optimizer):
        """Fence the stream ``optimizer.step()`` runs on before every step (``register_step_pre_hook``); returns the hook's
        handle."""
        return optimizer.register_step_pre_hook(lambda opt, args, kwargs: self.fence())

    def warmup(self, state_dict) -> int:
        """Optional (new): pay the one-time costs of the first ``async_save`` of ``state_dict`` now -- device staging buffer,
        pinned host slots (prefault + ``cudaHostRegister``: seconds for 16 GB), the plan with its tile tables -- instead of
        inside the first checkpoint of the training run.  Nothing is saved.  Returns the packed snapshot size in bytes."""
        tensors = []
        _collect_tensors(state_dict, tensors)
        cuda = [t for t in tensors if t.is_cuda]
        if not cuda:
            return 0
        from ..b200.engine import SnapshotEngine
        from ..b200.fastsave import zero_copy_enabled

        engine = SnapshotEngine.get(cuda[0].device.index)
        cuda = [t if t.is_contiguous() else t.contiguous() for t in cuda]
        container = zero_copy_enabled() and len(cuda) == len(tensors)
        plan = engine._plan_for(cuda, engine._narrow_mask(cuda, self._narrow), container)
        engine.reserve(plan.staging_bytes, len(cuda), staging=not self._direct)
        return plan.staging_bytes

    def load(self, f, map_location=None, *, into=None, strict: bool = True, verify: bool = False):
        """Load a ``torch.save`` file (new; ``async_save``'s files or any other).

        * ``map_location`` None or the CPU (and no ``into``): exactly ``torch.load(f, map_location=map_location)``.
        * ``map_location`` a CUDA device of this process (``"cuda"``, ``"cuda:k"``, ``torch.device``): what
          ``torch.load(f, map_location=that device)`` returns -- same dtypes, shapes, strides, storage offsets, bytes and
          storage sharing, one CUDA storage per file record -- read by the snapshot engine (parallel ``pread`` -> pinned
          ring -> HBM -> one scatter kernel; in place when ``f`` is a hard link to one of this process's pinned slots).
        * ``into=state_dict`` of live CUDA tensors (``map_location`` None): the saved bytes are written into those tensors
          where they are, matched by nested key path, any strides, fp32 / bf16 / fp16 converted on the device like
          ``target.copy_(saved)``; other dtype pairs and targets on the CPU or another device are copied with ``copy_``.
          ``strict=True`` raises on missing or unexpected keys before anything is read; shape mismatches always raise.
          Returns ``(missing_keys, unexpected_keys)`` like ``load_state_dict``.
        * ``verify=True``: every record read is checked against its CRC-32 field (on the GPU, over the bytes that reached
          HBM); a mismatch raises ``SnapError("crc32 mismatch ...")`` naming the key, the file and the record offset.
          In-place targets may hold the unverified bytes by then.  Records written without a CRC-32 are counted as
          unverified with one warning.

        The engine modes need a CUDA device and the engine library (``SnapError`` otherwise) and a path (or a file object
        opened on one).  ``SnapshotEngine.last_torch_load`` describes the last such load."""
        from ..b200.fastload import load

        if into is not None:
            self.fence()  # the load writes the live tensors a staging-free save may still be reading
        return load(f, map_location, into=into, strict=strict, verify=verify)

    def _reap(self, finalized=None):
        """Release the host slots of finalized calls."""
        if finalized is None:
            finalized = self._async_calls_queue.maybe_finalize_async_calls(blocking=False, no_dist=True)
        failed = None
        for idx in finalized:
            check = self._checks.pop(idx, None)
            if check is not None:
                try:
                    self.last_fence_check = check.verify()
                except Exception as e:  # noqa: BLE001 - raised once every finalized slot is released
                    failed = failed or e
            snap = self._pending.pop(idx, None)
            if snap is not None:
                snap.release()
        if self._pending and self._async_calls_queue.get_num_unfinalized_calls() == 0:
            # calls that were aborted (queue closed with abort=True) never finalize: free their slots
            for snap in self._pending.values():
                snap.release()
            self._pending.clear()
            self._checks.clear()
        self._unfenced = [s for s in self._unfenced if not s.released]
        if failed is not None:
            raise failed

    def finalize_async_save(self, blocking: bool = False, no_dist=True, terminate=False):
        """Finalize finished saves (all of them, waiting, if ``blocking``).  ``no_dist=True`` checks only this
        rank's writer; ``terminate=True`` closes the queue afterwards."""
        if blocking and self._async_calls_queue.get_num_unfinalized_calls() > 0:
            if not torch.distributed.is_initialized() or torch.distributed.get_rank() == 0:
                logger.info("Unfinalized async checkpoint saves. Finalizing them synchronously now.")
        self._reap(self._async_calls_queue.maybe_finalize_async_calls(blocking, no_dist=no_dist))
        if terminate:
            self._async_calls_queue.close()

    def _get_async_calls_queue(self):
        """Test hook: the underlying queue."""
        return self._async_calls_queue

    def close(self, abort=False):
        """Wait for outstanding saves and stop the writer (``abort`` is accepted for API compatibility and,
        like in the reference, not forwarded)."""
        if self._async_calls_queue is not None:
            self._async_calls_queue.close()
            for snap in self._pending.values():
                snap.release()
            self._pending.clear()
            self._checks.clear()
            self._unfenced = []

    def __del__(self):
        try:
            self.close()
        except Exception:  # noqa: BLE001
            pass


def _cuda_names(state_dict):
    """Dotted key paths of the CUDA tensors of ``state_dict``, in ``_walk_tensors`` order (dicts and lists)."""
    out = []

    def walk(x, path):
        if isinstance(x, torch.Tensor):
            if x.is_cuda:
                out.append(".".join(str(p) for p in path))
        elif isinstance(x, dict):
            for k, v in x.items():
                walk(v, path + (k,))
        elif isinstance(x, list):
            for k, v in enumerate(x):
                walk(v, path + (k,))

    walk(state_dict, ())
    return out


class _FenceCheck:
    """``check_fence`` of one staging-free save: the CRC-32s of its bit-copied tensors as the fenced stream saw them,
    compared with the written file's records at finalize."""

    def __init__(self, path, names, tensors, snap):
        self.path = path
        layout = snap.layout
        # bit copies of the caller's own tensors; a narrowed record differs from its tensor, and the copies of a
        # non-contiguous tensor read a temporary that no later write reaches
        self.items, self.unchecked = [], 0
        for name, t, src, dt, sdt in zip(names, tensors, snap.sources, layout.dtypes, layout.src_dtypes):
            if not t.nbytes:
                continue
            if dt == sdt and src.data_ptr() == t.data_ptr():
                self.items.append((name, t))
            else:
                self.unchecked += 1
        self.crcs = None
        self.done = None
        self._plan = None

    def run(self, stream) -> None:
        from ..b200.engine import CrcxPlan

        self.crcs = torch.zeros(max(len(self.items), 1), dtype=torch.int32).pin_memory()
        self.done = torch.cuda.Event()
        if self.items:
            ptrs = [t.data_ptr() for _, t in self.items]
            base = min(ptrs) & ~15
            self._plan = CrcxPlan([p - base for p in ptrs], [t.nbytes for _, t in self.items], self.items[0][1].get_device())
            self._plan.run(base, self.crcs.data_ptr(), stream.cuda_stream)
        self.done.record(stream)

    def verify(self) -> dict:
        from ..b200._cabi import E_STATE, SnapError
        from ..b200.fastload import key_name, plan_archive

        stats = {"path": str(self.path), "checked": 0, "unchecked": self.unchecked + (len(self.items) if self.crcs is None else 0)}
        if self.crcs is None:
            return stats
        self.done.synchronize()
        got = {name: int(c) & 0xFFFFFFFF for (name, _), c in zip(self.items, self.crcs.tolist())}
        plan = plan_archive(self.path)
        records = {key_name(e.path): plan.storages[e.storage].crc32 for e in plan.entries}
        bad = [name for name in got if records.get(name) != got[name]]
        self._plan = None
        stats["checked"] = len(got)
        if bad:
            raise SnapError(
                E_STATE, "check_fence",
                f"{len(bad)} saved tensor(s) changed between async_save and fence(): {bad} (file {self.path})",
            )
        return stats
