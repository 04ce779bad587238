"""Host snapshot buffers and the parallel checkpoint writer, CPU only (no CUDA calls: pin=False)."""
import os
import threading
import time
import zlib
from pathlib import Path

import numpy as np
import pytest
import torch


def make_hb(nbytes, name=None):
    from nvidia_resiliency_ext.checkpointing.b200.engine import HostBuffer

    return HostBuffer.create(nbytes, name=name, pin=False, prefault_threads=2)


def test_hostbuf_create_open_wait_crc(built_library):
    from nvidia_resiliency_ext.checkpointing.b200._cabi import SnapError
    from nvidia_resiliency_ext.checkpointing.b200.engine import HostBuffer

    name = f"/nvrx_test_{os.getpid()}"
    hb = make_hb(3_000_000, name)
    assert hb.capacity >= 3_000_000 and hb.data_ptr % 4096 == 0 and hb.progress == 0
    buf = hb.as_tensor(3_000_000)
    rng = np.random.default_rng(0)
    payload = rng.integers(0, 256, 3_000_000, dtype=np.uint8)
    buf.numpy()[:] = payload
    # crc32 in parallel pieces + combine == zlib
    for off, n, thr in ((0, 3_000_000, 1), (0, 3_000_000, 7), (13, 2_999_000, 3), (5, 0, 4), (100, 17, 16)):
        assert hb.crc32(off, n, thr) == zlib.crc32(payload[off : off + n].tobytes())
    # a second mapping (what a writer process does) sees the same bytes and the progress word
    other = HostBuffer.open(name)
    assert other.capacity == hb.capacity
    assert np.array_equal(other.as_tensor(1000).numpy(), payload[:1000])
    with pytest.raises(SnapError):
        other.wait(1, timeout_ms=50)  # nothing drained yet -> timeout
    import ctypes as C

    def drain_later():
        time.sleep(0.1)
        C.c_uint64.from_address(hb.progress_ptr).value = 42

    t = threading.Thread(target=drain_later)
    t.start()
    other.wait(42, timeout_ms=5000)
    t.join()
    assert other.progress == 42
    other.close()
    with pytest.raises(SnapError):
        HostBuffer.open("/nvrx_test_does_not_exist")
    hb.close()
    with pytest.raises(SnapError):
        HostBuffer.open(name)  # unlinked by the owner


def test_segment_views_have_own_storage_and_save(built_library, tmp_path):
    hb = make_hb(1 << 20)
    a = hb.segment(0, 4000, torch.float32, (10, 100))
    b = hb.segment(4096, 800, torch.int64, (100,))
    a.copy_(torch.arange(1000, dtype=torch.float32).view(10, 100))
    b.copy_(torch.arange(100))
    assert a.untyped_storage().nbytes() == 4000 and b.untyped_storage().nbytes() == 800
    torch.save({"a": a, "b": b}, tmp_path / "x.pt")  # differently typed views of ONE storage would be refused
    x = torch.load(tmp_path / "x.pt")
    assert torch.equal(x["a"], a) and torch.equal(x["b"], b)
    del a, b
    hb.close()


@pytest.mark.parametrize("as_file_object", [False, True])
def test_parallel_writer_produces_a_plain_torch_checkpoint(built_library, tmp_path, as_file_object):
    from nvidia_resiliency_ext.checkpointing.b200 import fastsave

    hb = make_hb(64 << 20)
    g = torch.Generator().manual_seed(0)
    specs = [((1000, 1000), torch.float32), ((3,), torch.int64), ((0, 5), torch.float32), ((), torch.float32), ((4097,), torch.bfloat16),
             ((2048, 2048), torch.float32), ((77,), torch.uint8)]
    views, off = [], 0
    for shape, dt in specs:
        n = int(np.prod(shape)) * torch.empty((), dtype=dt).element_size()
        off = (off + 511) // 512 * 512
        v = hb.segment(off, n, dt, shape)
        if v.numel():
            src = torch.randn(shape, generator=g) * 100 if dt.is_floating_point else torch.randint(0, 200, shape, generator=g)
            v.copy_(src.to(dt))
        views.append(v)
        off += n
    foreign = torch.arange(10.0)  # a tensor that does not live in the slot
    obj = {"slot": views, "nested": {"f": foreign, "txt": "hello", "again": views[0]}, "n": 3}
    path = tmp_path / "fast.pt"
    with fastsave.slot_ranges([(hb.data_ptr, hb.capacity, hb)]):
        if as_file_object:
            with open(path, "bx") as fh:
                how = fastsave.save(obj, fh)
        else:
            how = fastsave.save(obj, path)
    assert how == "parallel"
    import zipfile

    with zipfile.ZipFile(path) as z:
        assert z.testzip() is None  # record checksums are on by default
    torch.save(obj, tmp_path / "stock.pt")
    fast, stock = torch.load(path), torch.load(tmp_path / "stock.pt")
    for a, b in zip(fast["slot"], stock["slot"]):
        assert a.dtype == b.dtype and a.shape == b.shape and (a.numel() == 0 or torch.equal(a.view(-1).view(torch.uint8), b.view(-1).view(torch.uint8)))
    assert torch.equal(fast["nested"]["f"], foreign) and fast["nested"]["txt"] == "hello" and fast["n"] == 3
    assert fast["nested"]["again"].data_ptr() == fast["slot"][0].data_ptr()  # shared storage preserved, as with stock torch.save
    # same container layout as stock torch.save: same records at the same offsets
    r1, r2 = torch._C.PyTorchFileReader(str(path)), torch._C.PyTorchFileReader(str(tmp_path / "stock.pt"))
    recs = sorted(r1.get_all_records())
    assert recs == sorted(r2.get_all_records())
    if not as_file_object:  # (a file object is archived under the generic name "archive": different header lengths)
        assert all(r1.get_record_offset(n) - r2.get_record_offset(n) == r1.get_record_offset("data/0") - r2.get_record_offset("data/0")
                   for n in recs if n.startswith("data/"))
    assert torch.equal(torch.load(path, mmap=True)["slot"][5], stock["slot"][5])
    # outside a slot context the stock writer is used
    assert fastsave.save(obj, tmp_path / "plain.pt") == "torch"
    del views, obj, fast, stock
    hb.close()


def _fake_snapshot(name):
    """A drained snapshot slot built by hand (no GPU): two tensors + descriptor as SnapshotEngine would produce."""
    import ctypes as C

    from nvidia_resiliency_ext.checkpointing.b200.engine import PackedLayout

    hb = make_hb(1 << 20, name)
    a = torch.arange(1000, dtype=torch.float32).view(10, 100)
    b = torch.arange(77, dtype=torch.int64)
    layout = PackedLayout(shapes=[(10, 100), (77,)], dtypes=["float32", "int64"], src_dtypes=["float32", "int64"], offsets=[0, 4096],
                          packed_nbytes=[4000, 616], total_bytes=4096 + 1024)
    hb.segment(0, 4000, torch.float32, (10, 100)).copy_(a)
    hb.segment(4096, 616, torch.int64, (77,)).copy_(b)
    C.c_uint64.from_address(hb.progress_ptr).value = layout.total_bytes  # "drain finished"
    desc = {"shm_name": name, "progress_target": layout.total_bytes, "layout": layout, "owner_pid": os.getpid(), "owner_base": hb.data_ptr}
    return hb, desc, a, b


def test_writer_side_of_a_snapshot_in_process_and_spawned(built_library, tmp_path):
    """What the persistent worker runs for TorchAsyncCheckpoint.async_save: map the slot by name, wait for the
    drain, persist -- here against a hand-made slot so it runs without a GPU."""
    import torch.multiprocessing as mp

    from nvidia_resiliency_ext.checkpointing.b200.persist import SnapshotRef, save_snapshot_with_torch

    name = f"/nvrx_test_w_{os.getpid()}"
    hb, desc, a, b = _fake_snapshot(name)
    skeleton = {"model": {"a": SnapshotRef(0)}, "opt": [SnapshotRef(1), "x"], "it": 9}
    save_snapshot_with_torch(skeleton, tmp_path / "inproc.pt", desc)
    got = torch.load(tmp_path / "inproc.pt")
    assert torch.equal(got["model"]["a"], a) and torch.equal(got["opt"][0], b) and got["opt"][1] == "x" and got["it"] == 9
    ctx = mp.get_context("spawn")
    p = ctx.Process(target=save_snapshot_with_torch, args=(skeleton, str(tmp_path / "spawned.pt"), desc))
    p.start()
    p.join(120)
    assert p.exitcode == 0
    got = torch.load(tmp_path / "spawned.pt")
    assert torch.equal(got["model"]["a"], a) and torch.equal(got["opt"][0], b)
    hb.close()


def test_parallel_gather_into_slot(built_library):
    hb = make_hb(8 << 20)
    g = torch.Generator().manual_seed(3)
    srcs = [torch.randint(0, 255, (n,), dtype=torch.uint8, generator=g) for n in (0, 1, 4097, 3_000_000, 5)]
    offs, cur = [], 0
    for t in srcs:
        cur = (cur + 511) // 512 * 512
        offs.append(cur)
        cur += t.numel()
    hb.gather([t.data_ptr() for t in srcs], [t.numel() for t in srcs], offs, threads=5)
    view = hb.as_tensor(cur)
    for t, off in zip(srcs, offs):
        assert torch.equal(view[off : off + t.numel()], t)
    from nvidia_resiliency_ext.checkpointing.b200._cabi import SnapError

    with pytest.raises(SnapError):
        hb.gather([srcs[3].data_ptr()], [3_000_000], [hb.capacity - 10], threads=2)  # would run past the slot
    del view
    hb.close()


def test_persistent_writer_keeps_slots_mapped(built_library, tmp_path, monkeypatch):
    """The persistent worker sets NVRX_B200_CACHE_SLOTS: the slot mapping is reused across checkpoints and stale ones
    (slot re-created under another name) are dropped."""
    from nvidia_resiliency_ext.checkpointing.b200 import persist
    from nvidia_resiliency_ext.checkpointing.b200.persist import SnapshotRef, save_snapshot_with_torch

    monkeypatch.setenv("NVRX_B200_CACHE_SLOTS", "1")
    persist._slot_cache.clear()
    name = f"/nvrx_test_c_{os.getpid()}"
    hb, desc, a, b = _fake_snapshot(name)
    skeleton = {"a": SnapshotRef(0), "b": SnapshotRef(1)}
    for i in range(2):
        save_snapshot_with_torch(skeleton, tmp_path / f"c{i}.pt", desc)
        got = torch.load(tmp_path / f"c{i}.pt")
        assert torch.equal(got["a"], a) and torch.equal(got["b"], b)
    assert list(persist._slot_cache) == [name]
    cached = persist._slot_cache[name]
    hb.close()  # owner re-creates the slot under a new name
    name2 = name + "_g2"
    hb2, desc2, a2, b2 = _fake_snapshot(name2)
    save_snapshot_with_torch(skeleton, tmp_path / "c2.pt", desc2)
    assert list(persist._slot_cache) == [name2]  # the stale mapping was closed and dropped
    assert torch.equal(torch.load(tmp_path / "c2.pt")["a"], a2)
    persist._slot_cache.pop(name2).close(unlink=False)
    hb2.close()


def test_readv_fd_fills_the_slot_from_a_file(built_library, tmp_path):
    """Restore-side mirror of writev_fd: file ranges land at the given payload offsets (parallel pread)."""
    from nvidia_resiliency_ext.checkpointing.b200._cabi import SnapError

    rng = np.random.default_rng(11)
    blob = rng.integers(0, 256, 40_000_000, dtype=np.uint8)
    path = tmp_path / "blob.bin"
    blob.tofile(path)
    hb = make_hb(48 << 20)
    try:
        file_offs = [0, 1_000_003, 17_000_000, 39_999_990]
        sizes = [1_000_000, 15_999_997, 20_000_000, 10]
        dst = [512, 2 << 20, 20 << 20, 47 << 20]
        fd = os.open(path, os.O_RDONLY)
        try:
            hb.readv_fd(dst, sizes, file_offs, fd, threads=5)
            got = hb.as_tensor(hb.capacity).numpy()
            for d, n, f in zip(dst, sizes, file_offs):
                assert np.array_equal(got[d : d + n], blob[f : f + n])
            with pytest.raises(SnapError):  # range beyond the end of the file
                hb.readv_fd([0], [100], [39_999_990], fd, threads=2)
            with pytest.raises(SnapError):  # destination outside the slot
                hb.readv_fd([hb.capacity - 5], [100], [0], fd, threads=2)
        finally:
            os.close(fd)
    finally:
        hb.close()


def test_writev_fd_with_preallocation(built_library, tmp_path, monkeypatch):
    """NVRX_B200_WRITE_FALLOCATE=1 (opt-in): same bytes in the file, destination pages allocated by one fallocate call."""
    monkeypatch.setenv("NVRX_B200_WRITE_FALLOCATE", "1")
    rng = np.random.default_rng(2)
    hb = make_hb(24 << 20)
    try:
        payload = rng.integers(0, 256, 24 << 20, dtype=np.uint8)
        hb.as_tensor(24 << 20).numpy()[:] = payload
        offs, sizes, file_offs = [0, 9 << 20, (20 << 20) + 3], [5 << 20, 10 << 20, 1000], [4096, 6 << 20, 17 << 20]
        for path in (tmp_path / "disk.bin", Path("/dev/shm") / f"nvrx_falloc_{os.getpid()}.bin"):
            fd = os.open(path, os.O_CREAT | os.O_RDWR | os.O_TRUNC, 0o644)
            try:
                hb.writev_fd(offs, sizes, file_offs, fd, threads=4)
                got = np.fromfile(path, dtype=np.uint8)
                for o, n, f in zip(offs, sizes, file_offs):
                    assert np.array_equal(got[f : f + n], payload[o : o + n])
            finally:
                os.close(fd)
                os.unlink(path)
    finally:
        hb.close()


def test_crc32_fold_and_batched_sums_match_zlib(built_library):
    """The carry-less-multiply CRC (csrc/crc32_fold.cpp) behind nvrx_hostbuf_crc32 / crc32v against zlib: every alignment,
    lengths around the 16 / 64-byte folding blocks and the 4 MiB piece boundary of the batched call."""
    import os
    import random
    import zlib

    import numpy as np

    from nvidia_resiliency_ext.checkpointing.b200.engine import HostBuffer

    n = 24 << 20
    hb = HostBuffer.create(n, name=f"/nvrx_crc_t_{os.getpid()}", pin=False, prefault_threads=2)
    try:
        arr = np.frombuffer((__import__("ctypes").c_uint8 * n).from_address(hb.data_ptr), dtype=np.uint8)
        arr[:] = np.random.default_rng(3).integers(0, 256, n, dtype=np.uint8)
        rnd = random.Random(5)
        lens = [0, 1, 15, 16, 17, 63, 64, 65, 79, 80, 127, 128, 129, 1000, 4095, 4096, 4097, (4 << 20) - 1, 4 << 20, (4 << 20) + 1, (9 << 20) + 7]
        offs, sizes = [], []
        for ln in lens * 3:
            off = rnd.randrange(0, n - ln)
            offs.append(off)
            sizes.append(ln)
            assert hb.crc32(off, ln, threads=1) == zlib.crc32(arr[off : off + ln].tobytes())
        for threads in (1, 5):
            got = hb.crc32v(offs, sizes, threads=threads)
            assert got == [zlib.crc32(arr[o : o + s].tobytes()) for o, s in zip(offs, sizes)]
        assert hb.crc32(0, n, threads=4) == zlib.crc32(arr.tobytes())
    finally:
        hb.close()


def test_fastsave_falls_back_before_writing_into_unnamed_targets(built_library, tmp_path):
    """ADVICE r1: a BytesIO / offset target must get a complete stock torch.save, not a payload-less container followed by an
    exception."""
    import io

    from nvidia_resiliency_ext.checkpointing.b200 import fastsave

    hb = make_hb(1 << 20)
    v = hb.segment(0, 4000, torch.float32, (1000,))
    v.copy_(torch.arange(1000.0))
    obj = {"v": v, "k": 1}
    with fastsave.slot_ranges([(hb.data_ptr, hb.capacity, hb)]):
        buf = io.BytesIO()
        assert fastsave.save(obj, buf) == "torch"
        buf.seek(0)
        assert torch.equal(torch.load(buf)["v"], torch.arange(1000.0))
        with open(tmp_path / "off.bin", "w+b") as fh:
            fh.write(b"x" * 100)
            assert fastsave.save(obj, fh) == "torch"
            fh.seek(100)
            assert torch.equal(torch.load(io.BytesIO(fh.read()))["v"], torch.arange(1000.0))
    del v
    hb.close()


def test_writer_reports_a_full_file_system_as_an_error(built_library, tmp_path):
    """ADVICE r1: the destination range is allocated before it is mapped, so "no space" is an errno (NVRX_E_SYS), not a SIGBUS
    in the writer process.  A file limit (RLIMIT_FSIZE) stands in for the full disk."""
    import resource
    import signal

    from nvidia_resiliency_ext.checkpointing.b200._cabi import SnapError

    hb = make_hb(8 << 20)
    path = tmp_path / "limited.bin"
    old = resource.getrlimit(resource.RLIMIT_FSIZE)
    old_handler = signal.signal(signal.SIGXFSZ, signal.SIG_IGN)
    fd = os.open(path, os.O_CREAT | os.O_RDWR, 0o644)
    try:
        resource.setrlimit(resource.RLIMIT_FSIZE, (1 << 20, old[1]))
        with pytest.raises(SnapError) as exc:
            hb.writev_fd([0], [8 << 20], [0], fd, threads=2)
        assert exc.value.status == 1003  # NVRX_E_SYS with errno EFBIG
    finally:
        resource.setrlimit(resource.RLIMIT_FSIZE, old)
        signal.signal(signal.SIGXFSZ, old_handler)
        os.close(fd)
        hb.close()


def _save_repeatedly(path, seed, rounds):
    from nvidia_resiliency_ext.checkpointing.b200 import fastsave
    from nvidia_resiliency_ext.checkpointing.b200.engine import HostBuffer

    hb = HostBuffer.create(8 << 20, name=f"/nvrx_race_{os.getpid()}", pin=False, prefault_threads=1)
    try:
        v = hb.segment(0, 4 << 20, torch.float32, (1 << 20,))
        v.fill_(float(seed))
        with fastsave.slot_ranges([(hb.data_ptr, hb.capacity, hb)]):
            for _ in range(rounds):
                assert fastsave.save({"v": v, "who": seed}, path) == "parallel"
        del v
    finally:
        hb.close()


def test_several_writers_on_one_path_do_not_hurt_each_other(built_library, tmp_path):
    """The reference's own test saves the same path from every rank (tests/checkpointing/unit/test_async_save.py:38).  A writer
    that truncates the file another one has mapped kills that one with SIGBUS (seen at world size 2 on a GPU box): every
    writer fills a private file and renames it into place."""
    import multiprocessing as mp

    path = tmp_path / "shared.pt"
    ctx = mp.get_context("spawn")  # (fork of this multi-threaded test process + OpenMP in the child does not end well)
    procs = [ctx.Process(target=_save_repeatedly, args=(path, seed, 6)) for seed in (1, 2, 3)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(120)
    assert [p.exitcode for p in procs] == [0, 0, 0]
    got = torch.load(path)
    assert got["who"] in (1, 2, 3) and torch.all(got["v"] == float(got["who"]))  # one writer's complete file, not a mix
    assert sorted(x.name for x in tmp_path.iterdir()) == ["shared.pt"]  # no scratch directories left behind
