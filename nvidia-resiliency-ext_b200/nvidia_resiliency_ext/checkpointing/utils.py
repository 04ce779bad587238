"""Shared helpers of the checkpointing package.

Mirror of the reference module ``checkpointing/utils.py`` (same public names) with ``preload_tensors``
rebuilt on the H100 snapshot engine:

* ``preload_tensors``      reference ``utils.py:85-99``   -> one pack kernel + one side-stream drain
* ``debug_time`` & friends reference ``utils.py:34-82``   -> same log format ("<stack> took X.XXXXs"), the
  reference tests grep it (``tests/checkpointing/unit/test_cleanup.py:77-86``)
* ``_disable_gc``, ``wrap_for_async``, ``diff``, ``dict_list_map_outplace``  reference ``utils.py:102-192``
"""

from __future__ import annotations

import gc
import logging
import time
from contextlib import contextmanager
from typing import Any, Callable, Dict, List, Optional, Tuple, TypeVar, Union

import numpy as np
import torch

U = TypeVar("U")
V = TypeVar("V")

fallback_logger = logging.getLogger(__name__)

# (names, loggers) of the enclosing debug_time scopes; innermost last
_scope_names: List[str] = []
_scope_loggers: List[logging.Logger] = []


@contextmanager
def logger_stack(name: Optional[str] = None, current_logger: Optional[logging.Logger] = None):
    """Push a scope name / logger; yields ``(dotted scope path, logger to use)``."""
    pushed_name = bool(name)
    pushed_logger = current_logger is not None
    if pushed_name:
        _scope_names.append(name)
    if pushed_logger:
        _scope_loggers.append(current_logger)
    active = current_logger or (_scope_loggers[-1] if _scope_loggers else fallback_logger)
    try:
        yield ".".join(_scope_names), active
    finally:
        if pushed_name and _scope_names:
            _scope_names.pop()
        if pushed_logger and _scope_loggers:
            _scope_loggers.pop()


@contextmanager
def debug_time(
    name: str, logger: Optional[logging.Logger] = None, threshold: float = float("-inf"), level=None
):
    """Time a block and log ``"<scope path> took <seconds>s"``.

    Without ``threshold`` the message is DEBUG; with one it is WARNING and only emitted when the block took
    at least ``threshold`` seconds.  ``logger=None`` inherits the innermost enclosing scope's logger."""
    with logger_stack(name, logger) as (path, log):
        t0 = time.time()
        try:
            yield
        finally:
            elapsed = time.time() - t0
            if elapsed >= threshold:
                lvl = level
                if lvl is None:
                    lvl = logging.DEBUG if threshold == float("-inf") else logging.WARNING
                log.log(lvl, f"{path} took {elapsed:.4f}s")


def debug_msg(msg: str):
    with logger_stack(None, None) as (path, log):
        log.debug(f"{path} {msg}")


def dict_list_map_outplace(f: Callable[[U], V], x: Union[Dict, List, U]) -> Union[Dict, List, V]:
    """Rebuild a nested dict/list structure applying ``f`` to every leaf (input is left untouched)."""
    if isinstance(x, dict):
        return {k: dict_list_map_outplace(f, v) for k, v in x.items()}
    if isinstance(x, list):
        return [dict_list_map_outplace(f, v) for v in x]
    return f(x)


def _collect_tensors(x, out: list) -> None:
    if isinstance(x, dict):
        for v in x.values():
            _collect_tensors(v, out)
    elif isinstance(x, list):
        for v in x:
            _collect_tensors(v, out)
    elif isinstance(x, torch.Tensor):
        out.append(x)


def preload_tensors(state_dict: Dict, non_blocking=True, *, narrow: bool = False, return_snapshot: bool = False):
    """Stage every tensor of ``state_dict`` in host memory; returns a new dict with CPU tensors.

    Reference semantics (``utils.py:85-99``): out-of-place map, ``tensor.detach().to("cpu", non_blocking)``
    per tensor, non-tensors pass through.  Here all CUDA tensors are packed by ONE kernel into a device
    staging buffer which a side stream drains into ONE pinned shared-memory buffer; the returned CPU
    tensors are views into that buffer.

    ``non_blocking=True``  the views become valid when the drain finishes (``snapshot.wait()``), exactly as
                           the reference's copies are only valid after ``torch.cuda.synchronize()``.
    ``non_blocking=False`` waits for the drain (event wait, not a device-wide sync) before returning.
    ``narrow=True``        (new, opt-in) fp32 tensors are stored as bf16 (round-to-nearest-even).

    Lifetime: the returned tensors are views of a pooled pinned slot.  With ``return_snapshot=True`` the caller owns the
    handle (``snapshot.release()`` when done); otherwise the slot is released when the last returned tensor is collected.

    State dicts without CUDA tensors are returned as an out-of-place copy of the structure without touching
    the engine (this is the reference's CPU-only case, BASELINE config C1).
    """
    tensors: List[torch.Tensor] = []
    _collect_tensors(state_dict, tensors)
    if not any(t.is_cuda for t in tensors):
        out = dict_list_map_outplace(lambda v: v.detach() if isinstance(v, torch.Tensor) else v, state_dict)
        return (out, None) if return_snapshot else out

    from .b200.engine import SnapshotEngine

    devices = {t.device.index for t in tensors if t.is_cuda}
    if len(devices) != 1:
        raise ValueError(f"preload_tensors: tensors live on several CUDA devices {sorted(devices)}")
    snap = SnapshotEngine.get(devices.pop()).snapshot(tensors, narrow=narrow)
    host = snap.host_views()
    if not return_snapshot:
        # nobody else holds the Snapshot: the pinned slot stays reserved exactly as long as one of the returned views is alive
        # (the reference hands out tensors the caller owns; here they are windows into a pooled slot, which must neither be
        # reused under them nor stay reserved after them)
        keepalive = _ReleaseWithLastView(snap)
        for v in host:
            if isinstance(v, torch.Tensor) and not v.is_cuda:
                v._nvrx_slot_keepalive = keepalive
    views = iter(host)
    out = dict_list_map_outplace(lambda v: next(views) if isinstance(v, torch.Tensor) else v, state_dict)
    if not non_blocking:
        snap.wait()
    return (out, snap) if return_snapshot else out


class _ReleaseWithLastView:
    """Referenced by every host view of a snapshot; releases the snapshot's slot when the last of them is collected."""

    def __init__(self, snap):
        self._snap = snap

    def __del__(self):
        try:
            self._snap.release()
        except Exception:  # noqa: BLE001 - interpreter shutdown
            pass


@contextmanager
def _disable_gc():
    """Keep the garbage collector off inside the block (fork children / writers must not run finalizers)."""
    was_on = gc.isenabled()
    if was_on:
        gc.disable()
    try:
        yield
    finally:
        if was_on:
            gc.enable()


def wrap_for_async(fn):
    """Wrap a save function so it runs with GC disabled in the forked writer."""

    def wrapped(state_dict, *args, **kwargs):
        with _disable_gc():
            fn(state_dict, *args, **kwargs)

    return wrapped


def diff(x1: Any, x2: Any, prefix: Tuple = ()) -> Tuple[list, list, list]:
    """Recursive comparison of two nested dict/list structures.

    Returns ``(only_left, only_right, mismatch)``: key paths present on one side only, and
    ``(path, type_left, type_right)`` for leaves that differ (tensors compare element-wise)."""
    only_left: list = []
    only_right: list = []
    mismatch: list = []
    if isinstance(x1, dict) and isinstance(x2, dict):
        only_left = [prefix + (k,) for k in x1.keys() - x2.keys()]
        only_right = [prefix + (k,) for k in x2.keys() - x1.keys()]
        for k in x2.keys() & x1.keys():
            l, r, m = diff(x1[k], x2[k], prefix + (k,))
            only_left += l
            only_right += r
            mismatch += m
        return only_left, only_right, mismatch
    if isinstance(x1, (list, tuple, np.ndarray)):
        assert isinstance(x1, type(x2))
        extra = list(range(len(x1) - 1, len(x2) - 1, -1))
        only_left, only_right = list(extra), list(extra)
        for i, (a, b) in enumerate(zip(x1, x2)):
            l, r, m = diff(a, b, prefix + (i,))
            only_left += l
            only_right += r
            mismatch += m
        return only_left, only_right, mismatch
    if isinstance(x1, torch.Tensor) and isinstance(x2, torch.Tensor):
        if x1.device != x2.device:
            differs = not torch.all(x1.cpu() == x2.cpu())
        else:
            differs = not torch.all(x1 == x2)
    elif hasattr(x1, "replica_id") and hasattr(x2, "replica_id"):
        assert isinstance(x1, type(x2))
        return diff(x1.data, x2.data, prefix + (type(x1),))
    else:
        try:
            differs = bool(x1 != x2)
        except RuntimeError:
            differs = True
    if differs:
        mismatch.append((prefix, type(x1), type(x2)))
    return only_left, only_right, mismatch
