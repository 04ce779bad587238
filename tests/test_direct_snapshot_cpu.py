"""Staging-free snapshots (``TorchAsyncCheckpoint(device_staging=False)``, ``SnapshotEngine.snapshot(direct=True)``) without a
GPU: the schedule ``nvrx_direct_schedule`` makes with the real library, the argument checks of ``nvrx_snapshot_direct``
(they run before any CUDA call), and the engine's and the checkpoint's Python end to end against the device stand-in of
tests/_fake_device.py, extended here with the staging-free call."""
import ctypes as C
import os
import random
import weakref

import pytest
import torch

from _fake_device import FakeCudaTensor, FakeDeviceLib, _val, fake_device, plain

MiB = 1 << 20


# ---------------------------------------------------------------------------------------------------------------------
# the schedule, real library
# ---------------------------------------------------------------------------------------------------------------------
def _schedule(nbytes, flags, offsets, small, chunk):
    from nvidia_resiliency_ext.checkpointing.b200 import _cabi
    from nvidia_resiliency_ext.checkpointing.b200.engine import _u32_array, _u64_array

    n = len(nbytes)
    in_kernel, after = (C.c_uint8 * max(n, 1))(), (C.c_uint64 * max(n, 1))()
    rc = _cabi.lib().nvrx_direct_schedule(n, _u64_array(nbytes), _u32_array(flags), _u64_array(offsets), small, chunk,
                                           in_kernel, after)
    return rc, [in_kernel[i] for i in range(n)], [after[i] for i in range(n)]


def _layouts():
    """Segment sizes around the threshold, 4-byte scalars, empty and narrowed segments; dense and container offsets."""
    from nvidia_resiliency_ext.checkpointing.b200 import ptzip
    from nvidia_resiliency_ext.checkpointing.b200.engine import DIRECT_SMALL_BYTES, expected_layout

    rng = random.Random(7)
    t = DIRECT_SMALL_BYTES
    for case in range(12):
        sizes = [rng.choice([0, 4, 16, t - 4, t, t + 4, 3 * t, 5 * MiB + 12, rng.randrange(1, 3 * MiB) * 4]) for _ in range(60)]
        narrow = [bool(s) and rng.random() < (0.3 if case % 3 == 0 else 0.0) for s in sizes]
        packed = [s // 2 if nr else s for s, nr in zip(sizes, narrow)]
        if case % 2:
            offs, span = ptzip.slot_offsets(packed)
            total = -(-span // 512) * 512
        else:
            offs, _, total = expected_layout(sizes, narrow)
        yield sizes, [1 if nr else 0 for nr in narrow], offs, packed, total, rng.choice([1 * MiB, 4 * MiB, 64 * MiB])


def test_schedule_covers_every_byte_once_and_reports_in_order(built_library):
    from nvidia_resiliency_ext.checkpointing.b200.engine import DIRECT_SMALL_BYTES

    for sizes, flags, offs, packed, total, chunk in _layouts():
        rc, in_kernel, after = _schedule(sizes, flags, offs, DIRECT_SMALL_BYTES, chunk)
        assert rc == 0
        # the kernel subset: exactly the narrowed segments and the non-empty ones below the threshold
        assert [bool(k) for k in in_kernel] == [bool(p) and (bool(f) or s < DIRECT_SMALL_BYTES)
                                                 for s, f, p in zip(sizes, flags, packed)]
        copies = [i for i in range(len(sizes)) if not in_kernel[i] and packed[i]]
        # kernel subset + copy list cover every payload byte of the layout exactly once: the segments are disjoint ranges
        # inside the payload, so that is every non-empty segment in exactly one of the two
        kernel = [i for i in range(len(sizes)) if in_kernel[i]]
        assert sorted(kernel + copies) == [i for i, p in enumerate(packed) if p]
        assert all(offs[i] + packed[i] <= offs[i + 1] for i in range(len(offs) - 1)) and offs[-1] + packed[-1] <= total
        # copies in slot-offset order; the progress values rise, name the end of their copy, end at the total
        assert [offs[i] for i in copies] == sorted(offs[i] for i in copies)
        reports, group = [], 0
        for i in copies:
            group += packed[i]
            if after[i]:
                assert after[i] == offs[i] + packed[i], "a progress value past the end of its group"
                assert group >= chunk
                reports.append(after[i])
                group = 0
            else:
                assert group < chunk
        reports.append(total)  # nvrx_snapshot_direct's final report
        assert reports == sorted(reports) and reports[-1] == total
        assert all(after[i] == 0 for i in range(len(sizes)) if i not in copies)


def test_schedule_rejects_bad_layouts(built_library):
    from nvidia_resiliency_ext.checkpointing.b200 import _cabi

    assert _schedule([1024, 1024], [0, 0], [2048, 0], 64, MiB)[0] == _cabi.E_INVALID  # descending
    assert _schedule([1024, 1024], [0, 0], [0, 512], 64, MiB)[0] == _cabi.E_INVALID  # overlapping
    assert _schedule([1026], [1], [0], 64, MiB)[0] == _cabi.E_INVALID  # odd narrowed length


def test_snapshot_direct_rejects_bad_copy_lists(built_library):
    """Checked before any CUDA call: the progress word may never name a byte beyond a landed copy."""
    from nvidia_resiliency_ext.checkpointing.b200 import _cabi
    from nvidia_resiliency_ext.checkpointing.b200.engine import _ptr_array, _u64_array

    lib = _cabi.lib()
    buf = (C.c_uint8 * 8192)()
    host = C.addressof(buf)

    def call(dst, nb, after, total=8192):
        n = len(dst)
        return lib.nvrx_snapshot_direct(None, n, _ptr_array([0x1000] * n), _u64_array(dst), _u64_array(nb), _u64_array(after),
                                        host, total, None, 0, 0, None, None, None)

    assert call([1024, 0], [512, 512], [0, 0]) == _cabi.E_INVALID  # not in slot-offset order
    assert call([0, 1024], [512, 512], [600, 0]) == _cabi.E_INVALID  # report past the end of its copy
    assert call([0, 1024], [512, 512], [512, 500]) == _cabi.E_INVALID  # falling report
    assert call([0, 8000], [512, 512], [0, 0]) == _cabi.E_INVALID  # past the slot payload


# ---------------------------------------------------------------------------------------------------------------------
# the Python flow against the device stand-in
# ---------------------------------------------------------------------------------------------------------------------
class DirectFakeDeviceLib(FakeDeviceLib):
    """The stand-in plus ``nvrx_snapshot_direct``: the kernel plan packs into the slot at its own offsets, the copies are
    memmoves, and every progress report is remembered."""

    def __init__(self, real):
        super().__init__(real)
        self.progress_reports = []

    def nvrx_snapshot_direct(self, kernel, n, src, dst, nbytes, after, host, total, progress, base, device, start, stream, done):
        if _val(kernel):
            self.nvrx_pack(kernel, host, stream)  # offsets of the kernel plan are slot offsets
            self.calls.append("direct_kernel")
        reports = []
        for i in range(n):
            C.memmove(_val(host) + dst[i], src[i], nbytes[i])
            if after[i]:
                reports.append(base + after[i])
        reports.append(base + total)
        if _val(progress):
            C.c_uint64.from_address(_val(progress)).value = base + total
        self.progress_reports.append(reports)
        self.calls.append("direct")
        return 0


@pytest.fixture
def direct_device(monkeypatch, built_library):
    import _fake_device

    monkeypatch.setattr(_fake_device, "FakeDeviceLib", DirectFakeDeviceLib)
    with fake_device(monkeypatch) as (engine, lib):
        assert isinstance(lib, DirectFakeDeviceLib)
        waits = []
        from nvidia_resiliency_ext.checkpointing.b200 import engine as eng

        monkeypatch.setattr(eng, "stream_wait_event", lambda stream, ev: waits.append((stream, ev)))

        class _Stream:
            cuda_stream = 0

        monkeypatch.setattr(torch.cuda, "current_stream", lambda *a, **k: _Stream())
        yield engine, lib, waits


def _state(seed=0, wrap=True):
    from nvidia_resiliency_ext.checkpointing.b200.engine import DIRECT_SMALL_BYTES

    g = torch.Generator().manual_seed(seed)
    w = FakeCudaTensor.wrap if wrap else (lambda t: t)
    return {
        "model": {"w": w(torch.randn(700, 33, generator=g)), "norm": w(torch.randn(64, generator=g)),
                  "big": w(torch.randn(DIRECT_SMALL_BYTES // 4 + 3, generator=g)), "empty": w(torch.empty(0, 3))},
        "opt": [w(torch.tensor(2.5 + seed)), {"m": w(torch.randn(4097, generator=g).to(torch.bfloat16))}],
        "blob": w(torch.randint(0, 255, (300_001,), dtype=torch.uint8, generator=g)),
        "iteration": 12345 + seed,
    }


def _same(a, b):
    if isinstance(a, dict):
        assert list(a) == list(b)
        for k in a:
            _same(a[k], b[k])
    elif isinstance(a, list):
        assert len(a) == len(b)
        for x, y in zip(a, b):
            _same(x, y)
    elif isinstance(a, torch.Tensor):
        a, b = plain(a), plain(b)
        assert a.dtype == b.dtype and a.shape == b.shape
        assert a.numel() == 0 or torch.equal(a.contiguous().view(-1).view(torch.uint8), b.contiguous().view(-1).view(torch.uint8))
    else:
        assert a == b


@pytest.mark.parametrize("zero_copy", ["1", "0"])
def test_direct_saves_without_staging(monkeypatch, direct_device, shm_dir, dist_1rank, zero_copy):
    from nvidia_resiliency_ext.checkpointing.async_ckpt.torch_ckpt import TorchAsyncCheckpoint

    monkeypatch.setenv("NVRX_B200_ZERO_COPY", zero_copy)
    monkeypatch.setenv("NVRX_B200_GPU_CRC", "0")
    engine, lib, waits = direct_device
    engine.drain_chunk = 64 << 10  # several progress reports for this small state
    ckpt = TorchAsyncCheckpoint(persistent_queue=False, device_staging=False)
    try:
        assert ckpt.warmup(_state(0)) > 0 and engine._staging is None
        for i in range(3):
            sd = _state(i)
            sd["model"]["t"] = FakeCudaTensor.wrap(torch.randn(40, 30).t())  # non-contiguous: compacted
            want = _state(i, wrap=False)
            want["model"]["t"] = plain(sd["model"]["t"]).clone()
            path = shm_dir / f"d{i}.pt"
            ckpt.async_save(sd, path)
            snap = ckpt._pending[max(ckpt._pending)]
            assert snap.read_done is snap.slot.done_event
            temp = weakref.ref([s for s in snap.sources if plain(s).shape == (30, 40)][0])
            ckpt.fence()
            assert waits[-1][1] is snap.read_done
            ckpt.finalize_async_save(blocking=True)
            assert snap.released and snap.sources == [] and temp() is None  # held until release, not after
            _same(torch.load(path, weights_only=False), want)
            assert (os.stat(path).st_nlink == 2) == (zero_copy == "1")
        assert engine._staging is None
        assert "pack" in lib.calls and "direct_kernel" in lib.calls  # the small and 4-byte tensors
        assert "drain" not in lib.calls
        for reports in lib.progress_reports:
            assert reports == sorted(reports) and len(reports) > 1
    finally:
        ckpt.close()


def test_direct_narrowing_goes_through_the_kernel(monkeypatch, direct_device, tmp_path, dist_1rank):
    from nvidia_resiliency_ext.checkpointing.async_ckpt.torch_ckpt import TorchAsyncCheckpoint

    monkeypatch.setenv("NVRX_B200_GPU_CRC", "0")
    engine, lib, _ = direct_device
    ckpt = TorchAsyncCheckpoint(persistent_queue=False, device_staging=False, narrow_fp32_to_bf16=True)
    try:
        sd = _state(3)
        ckpt.async_save(sd, tmp_path / "n.pt")
        ckpt.finalize_async_save(blocking=True)
        got = torch.load(tmp_path / "n.pt", weights_only=False)
        assert torch.equal(got["model"]["big"], plain(sd["model"]["big"]).to(torch.bfloat16))
        assert torch.equal(got["blob"], plain(sd["blob"]))
        plan = engine._plans[next(iter(engine._plans))]
        kernel = plan.__dict__["_direct"]["kernel"]
        assert kernel is not None and list(kernel.offsets) == [plan.offsets[i] for i in plan.__dict__["_direct"]["small"]]
        assert engine._staging is None
    finally:
        ckpt.close()


def test_fence_is_a_no_op_in_the_default_mode(monkeypatch, direct_device, tmp_path, dist_1rank):
    from nvidia_resiliency_ext.checkpointing.async_ckpt.torch_ckpt import TorchAsyncCheckpoint

    monkeypatch.setenv("NVRX_B200_GPU_CRC", "0")
    engine, lib, waits = direct_device
    ckpt = TorchAsyncCheckpoint(persistent_queue=False)
    try:
        ckpt.fence()  # nothing saved yet
        ckpt.async_save(_state(1), tmp_path / "a.pt")
        n = len(waits)
        ckpt.fence()
        assert len(waits) == n and "direct" not in lib.calls
        ckpt.finalize_async_save(blocking=True)
    finally:
        ckpt.close()
    # staging-free, nothing pending: no wait either
    ckpt = TorchAsyncCheckpoint(persistent_queue=False, device_staging=False)
    try:
        ckpt.fence()
        assert len(waits) == n
    finally:
        ckpt.close()


def test_mode_errors(monkeypatch, built_library):
    from nvidia_resiliency_ext.checkpointing.async_ckpt.torch_ckpt import TorchAsyncCheckpoint

    monkeypatch.setenv("NVRX_B200_GPU_CRC", "1")
    with pytest.raises(ValueError, match="GPU_CRC"):
        TorchAsyncCheckpoint(device_staging=False)
    monkeypatch.setenv("NVRX_B200_GPU_CRC", "0")
    monkeypatch.setenv("NVRX_B200_ZIP_CRC", "0")
    with pytest.raises(ValueError, match="ZIP_CRC"):
        TorchAsyncCheckpoint(device_staging=False, check_fence=True)
    monkeypatch.setenv("NVRX_B200_ZIP_CRC", "1")
    with pytest.raises(ValueError, match="device_staging=False"):
        TorchAsyncCheckpoint(check_fence=True)


def test_engine_refuses_gpu_crc_for_direct_snapshots(monkeypatch, direct_device):
    engine, _, _ = direct_device
    monkeypatch.setenv("NVRX_B200_GPU_CRC", "1")
    with pytest.raises(ValueError, match="GPU_CRC"):
        engine.snapshot([FakeCudaTensor.wrap(torch.ones(8))], direct=True)


def test_fence_before_registers_a_step_pre_hook(monkeypatch, built_library):
    from nvidia_resiliency_ext.checkpointing.async_ckpt.torch_ckpt import TorchAsyncCheckpoint

    monkeypatch.setenv("NVRX_B200_GPU_CRC", "0")
    ckpt = TorchAsyncCheckpoint(persistent_queue=False, device_staging=False)
    try:
        fenced = []
        monkeypatch.setattr(ckpt, "fence", lambda stream=None: fenced.append(stream))
        p = torch.nn.Parameter(torch.ones(3))
        opt = torch.optim.SGD([p], lr=0.1)
        handle = ckpt.fence_before(opt)
        p.grad = torch.ones(3)
        opt.step()
        assert fenced == [None]
        handle.remove()
        opt.step()
        assert fenced == [None]
    finally:
        ckpt.close()
