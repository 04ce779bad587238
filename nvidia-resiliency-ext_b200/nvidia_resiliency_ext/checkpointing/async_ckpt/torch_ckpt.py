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

    def __init__(self, persistent_queue=True, *, narrow_fp32_to_bf16: bool = False):
        """``narrow_fp32_to_bf16`` (new, opt-in): store fp32 tensors as bf16 (halves drain + file size)."""
        self.save = torch.save
        self._async_calls_queue = AsyncCallsQueue(persistent=persistent_queue)
        self._narrow = narrow_fp32_to_bf16
        self._pending = {}  # call_idx -> Snapshot (host slot released on finalize)
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
        engine.reserve(plan.staging_bytes, len(cuda))
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

        return load(f, map_location, into=into, strict=strict, verify=verify)

    def _reap(self, finalized=None):
        """Release the host slots of finalized calls."""
        if finalized is None:
            finalized = self._async_calls_queue.maybe_finalize_async_calls(blocking=False, no_dist=True)
        for idx in finalized:
            snap = self._pending.pop(idx, None)
            if snap is not None:
                snap.release()
        if self._pending and self._async_calls_queue.get_num_unfinalized_calls() == 0:
            # calls that were aborted (queue closed with abort=True) never finalize: free their slots
            for snap in self._pending.values():
                snap.release()
            self._pending.clear()

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

    def __del__(self):
        try:
            self.close()
        except Exception:  # noqa: BLE001
            pass
