"""ctypes binding of ``libnvrx_snap.so`` (C ABI declared in ``include/nvrx_snap.h``).

The library is the product: there is deliberately NO Python/torch fallback here.  If the shared object is
missing or a call fails, :class:`SnapError` is raised -- the snapshot path never silently degrades to the
per-tensor ``tensor.to("cpu")`` loop of the reference (``checkpointing/utils.py:85-99``).
"""

from __future__ import annotations

import ctypes as C
import os
from pathlib import Path
from typing import Optional

ABI_VERSION = 2

OK = 0
E_INVALID = 1000
E_NOMEM = 1001
E_STATE = 1002
E_SYS = 1003
E_NODRIVER = 1004

SEG_NARROW_F32_BF16 = 0x1

VARIANT_AUTO = 0
VARIANT_LDG = 1
VARIANT_TMA = 2

# every symbol include/nvrx_snap.h declares; tests check the built library exports all of them
EXPORTED_SYMBOLS = (
    "nvrx_abi_version",
    "nvrx_strerror",
    "nvrx_device_info",
    "nvrx_plan_create",
    "nvrx_plan_create_at",
    "nvrx_plan_destroy",
    "nvrx_plan_info",
    "nvrx_plan_layout",
    "nvrx_plan_update_ptrs",
    "nvrx_plan_set_variant",
    "nvrx_plan_tiles",
    "nvrx_plan_commit",
    "nvrx_pack",
    "nvrx_scatter",
    "nvrx_pack_sharded",
    "nvrx_plan_set_shard_rotation",
    "nvrx_pack_broadcast",
    "nvrx_drain",
    "nvrx_snapshot",
    "nvrx_plan_last_launches",
    "nvrx_fill",
    "nvrx_fill_from_fd",
    "nvrx_dev_alloc",
    "nvrx_dev_free",
    "nvrx_stream_create",
    "nvrx_stream_destroy",
    "nvrx_event_create",
    "nvrx_event_destroy",
    "nvrx_event_record",
    "nvrx_stream_wait_event",
    "nvrx_event_query",
    "nvrx_event_sync",
    "nvrx_event_elapsed_ms",
    "nvrx_stream_sync",
    "nvrx_ipc_export",
    "nvrx_ipc_import",
    "nvrx_ipc_close",
    "nvrx_stream_write_u64",
    "nvrx_stream_wait_u64_geq",
    "nvrx_hostbuf_create",
    "nvrx_hostbuf_open",
    "nvrx_hostbuf_destroy",
    "nvrx_hostbuf_data",
    "nvrx_hostbuf_capacity",
    "nvrx_hostbuf_progress",
    "nvrx_hostbuf_wait",
    "nvrx_hostbuf_write_fd",
    "nvrx_hostbuf_writev_fd",
    "nvrx_hostbuf_gather",
    "nvrx_hostbuf_readv_fd",
    "nvrx_hostbuf_crc32",
    "nvrx_hostbuf_crc32v",
    "nvrx_crc_create",
    "nvrx_crc_destroy",
    "nvrx_crc_info",
    "nvrx_crc_run",
    "nvrx_crc_finish",
    "nvrx_crc_operator",
)


class SnapError(RuntimeError):
    """A C-ABI call returned a non-zero status (or the library is missing)."""

    def __init__(self, status: int, what: str, detail: str = ""):
        self.status = status
        msg = f"{what} failed with status {status}"
        if detail:
            msg += f" ({detail})"
        super().__init__(msg)


def library_path() -> Path:
    env = os.environ.get("NVRX_B200_LIB")
    if env:
        return Path(env)
    return Path(__file__).resolve().parent / "_lib" / "libnvrx_snap.so"


_LIB: Optional[C.CDLL] = None

_vp = C.c_void_p
_u64 = C.c_uint64
_i64 = C.c_int64
_u32 = C.c_uint32
_int = C.c_int


def _declare(lib: C.CDLL) -> None:
    P = C.POINTER
    sigs = {
        "nvrx_abi_version": (_int, []),
        "nvrx_strerror": (C.c_char_p, [_int]),
        "nvrx_device_info": (_int, [_int, P(_int), P(_u64), C.c_char_p, _int]),
        "nvrx_plan_create": (_int, [_i64, P(_vp), P(_u64), P(_u32), _u64, _u32, _int, P(_vp)]),
        "nvrx_plan_create_at": (_int, [_i64, P(_vp), P(_u64), P(_u32), P(_u64), _u64, _u32, _int, P(_vp)]),
        "nvrx_plan_destroy": (_int, [_vp]),
        "nvrx_plan_info": (_int, [_vp, P(_u64), P(_u64), P(_u64)]),
        "nvrx_plan_layout": (_int, [_vp, P(_u64), P(_u64)]),
        "nvrx_plan_update_ptrs": (_int, [_vp, P(_vp)]),
        "nvrx_plan_set_variant": (_int, [_vp, _int]),
        "nvrx_plan_tiles": (_int, [_vp, _u64, P(_u32), P(_u32), P(_u32), P(_u32), P(_u64), _u64]),
        "nvrx_plan_commit": (_int, [_vp, _vp]),
        "nvrx_pack": (_int, [_vp, _vp, _vp]),
        "nvrx_scatter": (_int, [_vp, _vp, _vp]),
        "nvrx_pack_sharded": (_int, [_vp, _vp, P(_vp), _int, _u64, _u64, _vp]),
        "nvrx_plan_set_shard_rotation": (_int, [_vp, _u32]),
        "nvrx_pack_broadcast": (_int, [_vp, P(_vp), _int, _u64, _vp]),
        "nvrx_drain": (_int, [_vp, _vp, _u64, _u64, _vp, _u64, _vp, _vp]),
        "nvrx_snapshot": (_int, [_vp, _vp, _vp, _u64, _vp, _u64, _vp, _vp, _vp, _vp]),
        "nvrx_plan_last_launches": (_int, [_vp, P(_u32)]),
        "nvrx_fill": (_int, [_vp, _vp, _u64, _u64, _vp, _vp]),
        "nvrx_fill_from_fd": (_int, [_vp, _u64, _int, _i64, P(_u64), P(_u64), P(_u64), _u64, _int, _int, _int, _vp]),
        "nvrx_dev_alloc": (_int, [_int, _u64, P(_vp)]),
        "nvrx_dev_free": (_int, [_int, _vp]),
        "nvrx_stream_create": (_int, [_int, _int, P(_vp)]),
        "nvrx_stream_destroy": (_int, [_vp]),
        "nvrx_event_create": (_int, [_int, _int, P(_vp)]),
        "nvrx_event_destroy": (_int, [_vp]),
        "nvrx_event_record": (_int, [_vp, _vp]),
        "nvrx_stream_wait_event": (_int, [_vp, _vp]),
        "nvrx_event_query": (_int, [_vp, P(_int)]),
        "nvrx_event_sync": (_int, [_vp]),
        "nvrx_event_elapsed_ms": (_int, [_vp, _vp, P(C.c_float)]),
        "nvrx_stream_sync": (_int, [_vp]),
        "nvrx_ipc_export": (_int, [_vp, C.c_char_p]),
        "nvrx_ipc_import": (_int, [_int, C.c_char_p, P(_vp)]),
        "nvrx_ipc_close": (_int, [_int, _vp]),
        "nvrx_stream_write_u64": (_int, [_vp, _vp, _u64]),
        "nvrx_stream_wait_u64_geq": (_int, [_vp, _vp, _u64]),
        "nvrx_hostbuf_create": (_int, [C.c_char_p, _u64, _int, _int, _int, P(_vp)]),
        "nvrx_hostbuf_open": (_int, [C.c_char_p, P(_vp)]),
        "nvrx_hostbuf_destroy": (_int, [_vp, _int]),
        "nvrx_hostbuf_data": (_vp, [_vp]),
        "nvrx_hostbuf_capacity": (_u64, [_vp]),
        "nvrx_hostbuf_progress": (_vp, [_vp]),
        "nvrx_hostbuf_wait": (_int, [_vp, _u64, _i64]),
        "nvrx_hostbuf_write_fd": (_int, [_vp, _u64, _u64, _int, _u64, _int]),
        "nvrx_hostbuf_writev_fd": (_int, [_vp, _i64, P(_u64), P(_u64), P(_u64), _int, _int]),
        "nvrx_hostbuf_gather": (_int, [_vp, _i64, P(_vp), P(_u64), P(_u64), _int]),
        "nvrx_hostbuf_readv_fd": (_int, [_vp, _i64, P(_u64), P(_u64), P(_u64), _int, _int]),
        "nvrx_hostbuf_crc32": (_int, [_vp, _u64, _u64, _int, P(_u32)]),
        "nvrx_hostbuf_crc32v": (_int, [_vp, _i64, P(_u64), P(_u64), _int, P(_u32)]),
        "nvrx_crc_create": (_int, [_i64, P(_u64), P(_u64), _int, P(_vp)]),
        "nvrx_crc_destroy": (_int, [_vp]),
        "nvrx_crc_info": (_int, [_vp, P(_u64)]),
        "nvrx_crc_run": (_int, [_vp, _vp, _vp, _vp, _u64, _vp]),
        "nvrx_crc_finish": (_int, [_i64, P(_u64), P(_u64), _vp, _u64, _vp, P(_u32)]),
        "nvrx_crc_operator": (_int, [_u32, P(_u32)]),
    }
    assert set(sigs) == set(EXPORTED_SYMBOLS)
    for name, (res, args) in sigs.items():
        fn = getattr(lib, name)
        fn.restype = res
        fn.argtypes = args


def lib() -> C.CDLL:
    """Load (once) and return the shared library; raises SnapError if it is missing."""
    global _LIB
    if _LIB is None:
        path = library_path()
        if not path.exists():
            raise SnapError(
                E_STATE,
                "loading libnvrx_snap.so",
                f"{path} not found - run `python -c 'import __graft_entry__ as g; g.build()'` "
                "(nvcc, sm_90a); there is no CPU fallback for the snapshot path",
            )
        handle = C.CDLL(str(path), use_errno=True)
        _declare(handle)
        got = handle.nvrx_abi_version()
        if got != ABI_VERSION:
            raise SnapError(E_STATE, "ABI check", f"library ABI {got} != binding ABI {ABI_VERSION}")
        _LIB = handle
    return _LIB


def strerror(status: int) -> str:
    return lib().nvrx_strerror(status).decode()


def check(status: int, what: str) -> None:
    if status != OK:
        detail = strerror(status)
        if status == E_SYS:
            err = C.get_errno()
            if err:
                detail += f": {os.strerror(err)}"
        raise SnapError(status, what, detail)
