"""TEST INFRASTRUCTURE: the box-scatter entry points on top of ``_fake_device``'s stand-in GPU, for the CPU tests of
``SnapshotEngine.load_boxes`` and ``CachedMetadataFileSystemReader(load_on_engine=True)``.

* ``nvrx_box_scatter`` replays the REAL planner's tile list (``nvrx_boxplan_tiles``) and row geometry
  (``nvrx_boxplan_box``) with memmoves, so the CPU tests exercise the tiles the kernel walks.
* ``nvrx_fill_from_fd`` behaves like the real pipeline where it matters for placement: the real one sends each pinned
  ring chunk to the device from the call's first to its last byte in that chunk, gaps between extents included.  Here the
  whole span of a call is first overwritten with a poison pattern, then the extents are read -- anything another call
  placed inside that span is destroyed, as it would be on the GPU.
* ``FakeCudaView`` stays a "CUDA tensor" through every view op (the DCP planner narrows targets)."""
import contextlib
import ctypes as C
import os
import types

import torch

from _fake_device import FakeCudaTensor, _val, fake_device


class FakeCudaView(FakeCudaTensor):
    """Like FakeCudaTensor, but every view of it (narrow, slicing, ...) still looks like a CUDA tensor of cuda:0."""

    @classmethod
    def __torch_function__(cls, func, types, args=(), kwargs=None):
        with torch._C.DisableTorchFunctionSubclass():
            out = func(*args, **(kwargs or {}))
        if isinstance(out, torch.Tensor) and not isinstance(out, FakeCudaView):
            return torch.Tensor._make_subclass(FakeCudaView, out.detach())
        return out


def fake_cuda(t: torch.Tensor) -> FakeCudaView:
    return torch.Tensor._make_subclass(FakeCudaView, t.detach())


def _box_scatter(self, h, staging, stream):
    n = C.c_uint64()
    assert self._real.nvrx_boxplan_tiles(h, C.byref(n), None, None, None, None, None, 0) == 0
    cnt = max(n.value, 1)
    box, nby = (C.c_uint32 * cnt)(), (C.c_uint32 * cnt)()
    row, nrows, off = (C.c_uint64 * cnt)(), (C.c_uint64 * cnt)(), (C.c_uint64 * cnt)()
    assert self._real.nvrx_boxplan_tiles(h, None, box, row, nrows, off, nby, n.value) == 0
    geo = {}
    for t in range(n.value):
        b = box[t]
        if b not in geo:
            rb, no, so, dst = C.c_uint64(), C.c_uint32(), C.c_uint64(), C.c_uint64()
            sz, ss, ds = (C.c_uint64 * 8)(), (C.c_int64 * 8)(), (C.c_int64 * 8)()
            assert self._real.nvrx_boxplan_box(h, b, C.byref(rb), C.byref(no), sz, ss, ds, C.byref(so), C.byref(dst)) == 0
            k = no.value
            geo[b] = (rb.value, list(sz)[:k], list(ss)[:k], list(ds)[:k], so.value, dst.value)
        rb, sz, ss, ds, so, dst = geo[b]
        for r in range(row[t], row[t] + nrows[t]):
            s_addr, d_addr, q = _val(staging) + so, dst, r
            for d in range(len(sz) - 1, -1, -1):
                q, i = divmod(q, sz[d])
                s_addr += i * ss[d]
                d_addr += i * ds[d]
            lo, length = (off[t], nby[t]) if nrows[t] == 1 else (0, rb)
            C.memmove(d_addr + lo, s_addr + lo, length)
    self.calls.append("box_scatter")
    return 0


def _fill_from_fd_with_gaps(self, staging, staging_bytes, fd, n, stg_offs, nbytes, file_offs, chunk, slots, threads, device, stream):
    live = [i for i in range(n) if nbytes[i]]
    if live:
        lo, hi = stg_offs[live[0]], stg_offs[live[-1]] + nbytes[live[-1]]
        assert hi <= staging_bytes
        C.memset(_val(staging) + lo, 0xA5, hi - lo)
    for i in live:
        data = os.pread(fd, nbytes[i], file_offs[i])
        assert len(data) == nbytes[i]
        C.memmove(_val(staging) + stg_offs[i], data, nbytes[i])
    self.calls.append("fill_from_fd")
    return 0


@contextlib.contextmanager
def fake_box_device(monkeypatch):
    """``fake_device`` plus the box-scatter entry points; yields ``(engine, lib)``."""
    with fake_device(monkeypatch) as (engine, lib):
        lib.nvrx_box_scatter = types.MethodType(_box_scatter, lib)
        lib.nvrx_boxplan_commit = lambda h, stream: 0
        lib.nvrx_fill_from_fd = types.MethodType(_fill_from_fd_with_gaps, lib)
        yield engine, lib
