"""The engine's hand-offs of its shared buffers, with the hazard window held open on one GPU.

``SnapshotEngine`` owns one device staging buffer and a pool of pinned shm slots, used by the pack (training stream), the
drain (``_side``), the GPU checksum (``_aux``), the restores, the file restore, ``load_boxes`` and staging growth.  A drain
of a test-sized state ends long before Python issues the next call, so without help a missing wait passes unnoticed.  Every
test here therefore puts a sleep kernel (``torch.cuda._sleep``, calibrated once per session, ending by itself) at the head
of ``_side`` or ``_aux`` just before the operation under test, and asserts that the held work was still pending when the
next operation was issued: without that assert a pass would prove nothing.

The references are plain data: clones taken right after each save (the live tensors are then changed on the training
stream), files read back with ``torch.load`` and ``zipfile``'s CRC check, and the stock ``FileSystemReader``.  Everything
is compared byte for byte.  Files are written by the copying writer (``NVRX_B200_ZERO_COPY=0``) so that slots are handed
back to the pool and reused."""
import threading
import time
import zipfile

import pytest
import torch

pytestmark = pytest.mark.gpu

MiB = 1 << 20
DRAIN_CHUNK = 16 * MiB  # 29 chunks per drain of the default state
# Covers a writer fork and the Python between two calls.  On a shared H100 host that Python alone took 100-180 ms for the
# DCP load and more than 250 ms for a file restore with checksums, which closed a 250 ms window now and then: the test then
# fails its own premise.  A second leaves several times that margin and costs about a second per held test.
HOLD_MS = 1000


# ---------------------------------------------------------------------------------------------------------------------
# the hold
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="session")
def cycles_per_ms(built_library, tmp_path_factory):
    """Sleep-kernel cycles per millisecond.  First, every kernel a held window launches runs once (the first launch of a
    kernel loads its module, which can wait for the sleeping kernel and close the window), and one file restore creates
    the process's pinned read ring (hundreds of milliseconds, which would otherwise close the window)."""
    from nvidia_resiliency_ext.checkpointing.b200 import ptzip
    from nvidia_resiliency_ext.checkpointing.b200.engine import SnapshotEngine

    torch.cuda.set_device(0)
    sd = make_state(0)
    narrowed(clone(sd))
    mutate(sd)
    with pytest.MonkeyPatch.context() as mp:
        mp.setenv("NVRX_B200_ZERO_COPY", "0")
        for timing in (False, True):
            eng = SnapshotEngine(0, drain_chunk=DRAIN_CHUNK, timing=timing)
            for narrow, crc in ((False, "0"), (True, "0"), (False, "1")):
                mp.setenv("NVRX_B200_GPU_CRC", crc)
                snap = eng.snapshot(list(sd.values()), narrow=narrow)
                snap.wait()
                snap.release()
            if not timing:
                path = tmp_path_factory.mktemp("warm_ring") / "w.pt"
                torch.save([torch.ones(1 << 20), torch.zeros(4096)], path)
                host = torch.load(path, mmap=True, weights_only=True)
                offs = ptzip.tensor_offsets_in_file(path, host)
                assert offs is not None
                restores = eng.file_restores
                eng.restore(host, file_source=(str(path), offs))
                assert eng.file_restores == restores + 1
            torch.cuda.synchronize()
            eng.close()
    del sd
    torch.cuda._sleep(1000)
    torch.cuda.synchronize()
    rates = []
    for _ in range(3):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        torch.cuda._sleep(20_000_000)
        b.record()
        b.synchronize()
        rates.append(20_000_000 / a.elapsed_time(b))
    return max(rates)  # the fastest clock seen: a hold lasts at least as long as asked


def _ext(handle: int) -> torch.cuda.ExternalStream:
    return torch.cuda.ExternalStream(handle, device=torch.device("cuda", 0))


def hold(handle: int, cycles_per_ms: float, ms: float = HOLD_MS) -> None:
    """Queue a sleep kernel on an engine stream: what is queued behind it cannot start for ``ms`` milliseconds."""
    with torch.cuda.stream(_ext(handle)):
        torch.cuda._sleep(int(cycles_per_ms * ms))


def queued_after(handle: int) -> torch.cuda.Event:
    """An event behind everything queued on an engine stream so far."""
    ev = torch.cuda.Event()
    ev.record(_ext(handle))
    return ev


def assert_open(ev: torch.cuda.Event) -> None:
    assert not ev.query(), "the held work finished before the next operation was issued: the window was closed"


def spy_entry(monkeypatch, eng, name: str, ev: torch.cuda.Event) -> list:
    """Wrap ``eng.<name>``: every call records whether ``ev`` had completed when it was entered."""
    seen, orig = [], getattr(eng, name)

    def wrapped(*args, **kwargs):
        seen.append(ev.query())
        return orig(*args, **kwargs)

    monkeypatch.setattr(eng, name, wrapped)
    return seen


# ---------------------------------------------------------------------------------------------------------------------
# state, references, engines
# ---------------------------------------------------------------------------------------------------------------------
def make_state(seed: int, n_big: int = 6, big=(4096, 4608)) -> dict:
    """~0.48 GB by default; ten tensors, so that ``torch.save`` numbers its records in file order."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    sd = {f"w{i}": torch.randn(big, device="cuda", generator=g) for i in range(n_big)}
    sd["odd"] = torch.randn(3001, 1031, device="cuda", generator=g)
    sd["half"] = torch.randn(4099, 777, device="cuda", generator=g).to(torch.bfloat16)
    sd["ids"] = torch.randint(-(1 << 40), 1 << 40, (1_000_003,), device="cuda", generator=g)
    sd["step"] = torch.tensor(float(seed) + 0.25, device="cuda")
    return sd


def clone(sd: dict) -> dict:
    return {k: v.clone() for k, v in sd.items()}


def mutate(sd: dict) -> None:
    """The next training step, on the training stream: every element of every tensor changes."""
    for v in sd.values():
        v.add_(1)


def narrowed(sd: dict) -> dict:
    return {k: v.to(torch.bfloat16) if v.dtype == torch.float32 else v for k, v in sd.items()}


def nbytes(sd: dict) -> int:
    return sum(v.numel() * v.element_size() for v in sd.values())


def _bytes(t: torch.Tensor) -> torch.Tensor:
    return t.detach().cpu().contiguous().reshape(-1).view(torch.uint8)


def assert_same(got: dict, want: dict, what: str) -> None:
    assert list(got) == list(want), what
    bad = {}
    for k in want:
        assert got[k].dtype == want[k].dtype and got[k].shape == want[k].shape, (what, k)
        n = int((_bytes(got[k]) != _bytes(want[k])).sum())
        if n:
            bad[k] = n
    assert not bad, f"{what}: {sum(bad.values())} of {nbytes(want)} bytes differ {bad}"


def assert_file(path, want: dict, crc_checked: bool = False) -> None:
    if crc_checked:
        with zipfile.ZipFile(path) as zf:
            assert zf.testzip() is None, f"{path}: a record fails its CRC-32"
    assert_same(torch.load(path, weights_only=False, mmap=True), want, str(path))


@pytest.fixture
def engines(monkeypatch, built_library):
    """Fresh engines (16 MiB drain chunks) installed as the device-0 singleton that the API classes use."""
    from nvidia_resiliency_ext.checkpointing.b200.engine import SnapshotEngine

    torch.cuda.set_device(0)
    monkeypatch.setenv("NVRX_B200_ZERO_COPY", "0")
    made = []

    def make(**kwargs):
        kwargs.setdefault("drain_chunk", DRAIN_CHUNK)
        eng = SnapshotEngine(0, **kwargs)
        monkeypatch.setitem(SnapshotEngine._instances, 0, eng)
        made.append(eng)
        return eng

    yield make
    torch.cuda.synchronize()
    for eng in made:
        eng.close()


@pytest.fixture
def ckpts(engines, shm_dir):
    """TorchAsyncCheckpoint objects with forked writers, warmed up by one small save (first imports and fork outside the
    held windows); finalized and closed before the engines go."""
    from nvidia_resiliency_ext.checkpointing.async_ckpt.torch_ckpt import TorchAsyncCheckpoint

    made = []

    def make(**kwargs):
        made.append(TorchAsyncCheckpoint(persistent_queue=False, **kwargs))
        made[-1].async_save({"warm": torch.ones(1024, device="cuda")}, shm_dir / "_warm.pt")
        made[-1].finalize_async_save(blocking=True)
        return made[-1]

    yield make
    for c in made:
        c.finalize_async_save(blocking=True)
        c.close()


def reserve(eng, sd: dict, narrow: bool = False, extra: int = 4 * MiB) -> int:
    """Staging and both slots for snapshots of ``sd`` (plus ``extra``, room for GPU checksum values): no allocation or
    pinning inside a held window.  Returns the packed size."""
    tensors = list(sd.values())
    plan = eng._plan_for(tensors, eng._narrow_mask(tensors, narrow), False)
    eng.reserve(plan.staging_bytes + extra)
    return plan.staging_bytes


def save(ckpt, sd: dict, path):
    """``async_save`` and the engine snapshot it took."""
    ckpt.async_save(sd, path)
    return ckpt._pending[max(ckpt._pending)]


# ---------------------------------------------------------------------------------------------------------------------
# 1. snapshot then snapshot
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", ["pipelined", "timing", "narrow"])
def test_snapshot_then_snapshot(engines, ckpts, shm_dir, cycles_per_ms, mode):
    """The second pack must wait for the first drain (``_staging_free``) before it overwrites staging."""
    eng = engines(timing=mode == "timing")
    narrow = mode == "narrow"
    ckpt = ckpts(narrow_fp32_to_bf16=narrow)
    sd = make_state(1)
    reserve(eng, sd, narrow)
    hold(eng._side.handle, cycles_per_ms)
    a = save(ckpt, sd, shm_dir / "a.pt")
    want_a = clone(sd)
    mutate(sd)
    assert not a.drained(), "the window was closed"
    b = save(ckpt, sd, shm_dir / "b.pt")
    want_b = clone(sd)
    mutate(sd)
    assert a.slot is not b.slot
    ckpt.finalize_async_save(blocking=True)
    fix = narrowed if narrow else (lambda x: x)
    assert_file(shm_dir / "a.pt", fix(want_a))
    assert_file(shm_dir / "b.pt", fix(want_b))


# ---------------------------------------------------------------------------------------------------------------------
# 2. snapshot then restore(), 3. snapshot then file restore, 4. snapshot then dcp.load on the engine
# ---------------------------------------------------------------------------------------------------------------------
def test_snapshot_then_restore(engines, ckpts, shm_dir, cycles_per_ms):
    """restore()'s H2D into staging must wait for the pending drain."""
    eng, ckpt = engines(), ckpts()
    sd = make_state(2)
    other = {k: v.cpu() for k, v in make_state(20).items()}
    reserve(eng, sd)
    hold(eng._side.handle, cycles_per_ms)
    a = save(ckpt, sd, shm_dir / "a.pt")
    want = clone(sd)
    mutate(sd)
    assert not a.drained(), "the window was closed"
    back = eng.restore(list(other.values()))
    assert_same(dict(zip(other, back)), other, "restored")
    ckpt.finalize_async_save(blocking=True)
    assert_file(shm_dir / "a.pt", want)


def test_snapshot_then_file_restore(engines, ckpts, shm_dir, cycles_per_ms, dist_1rank, monkeypatch):
    """LocalCheckpointManager.load() -> _restore_from_file: nvrx_fill_from_fd into staging must wait for the pending drain."""
    from nvidia_resiliency_ext.checkpointing.local.basic_state_dict import BasicTensorAwareStateDict
    from nvidia_resiliency_ext.checkpointing.local.ckpt_managers.local_manager import LocalCheckpointManager

    eng, ckpt = engines(), ckpts()
    sd = make_state(3)
    reserve(eng, sd)
    on_disk = make_state(30)
    want_disk = {k: v.cpu() for k, v in on_disk.items()}
    LocalCheckpointManager(shm_dir / "local").save(BasicTensorAwareStateDict(on_disk), 1, is_async=False)
    del on_disk
    mgr = LocalCheckpointManager(shm_dir / "local")
    assert mgr.find_latest() == 1  # (a collective: outside the window)
    restores = eng.file_restores
    hold(eng._side.handle, cycles_per_ms)
    save(ckpt, sd, shm_dir / "a.pt")
    want = clone(sd)
    mutate(sd)
    seen = spy_entry(monkeypatch, eng, "_restore_from_file", queued_after(eng._side.handle))
    loaded, _ = mgr.load()
    assert seen == [False], "the window was closed (or the file path was not taken)"
    assert eng.file_restores == restores + 1
    assert_same(dict(zip(want_disk, loaded.tensors)), want_disk, "loaded from file")
    ckpt.finalize_async_save(blocking=True)
    assert_file(shm_dir / "a.pt", want)


def _dcp_state():
    g = torch.Generator(device="cuda").manual_seed(4)
    return {
        "w": torch.randn(4096, 8192, device="cuda", generator=g),
        "t": torch.randn(2048, 4096, device="cuda", generator=g).t(),
        "b": torch.randn(4099, 777, device="cuda", generator=g).to(torch.bfloat16),
        "ids": torch.randint(0, 1 << 40, (333, 7), device="cuda", generator=g),
        "step": torch.tensor(7.0, device="cuda"),
    }


@pytest.fixture(scope="module")
def dcp_checkpoint(tmp_path_factory, built_library):
    import torch.distributed.checkpoint as dcp

    path = tmp_path_factory.mktemp("handoff_dcp") / "ck"
    dcp.save({k: v.cpu() for k, v in _dcp_state().items()}, checkpoint_id=str(path))
    return path


@pytest.mark.parametrize("verify,staging_mb", [(False, 0), (True, 0), (True, 64)])
def test_snapshot_then_dcp_load(engines, ckpts, shm_dir, cycles_per_ms, dcp_checkpoint, monkeypatch, verify, staging_mb):
    """load_boxes' fills into staging must wait for the pending drain, every batch of them."""
    import torch.distributed.checkpoint as dcp
    from torch.distributed.checkpoint import FileSystemReader

    from nvidia_resiliency_ext.checkpointing.async_ckpt.cached_metadata_filesystem_reader import CachedMetadataFileSystemReader
    from nvidia_resiliency_ext.checkpointing.b200.engine import SnapshotEngine

    if staging_mb:
        monkeypatch.setattr(SnapshotEngine, "DCP_LOAD_STAGING", staging_mb * MiB)
    eng, ckpt = engines(), ckpts()
    sd = make_state(5)
    reserve(eng, sd)
    like = _dcp_state()
    ref = {k: torch.zeros_like(v) for k, v in like.items()}
    dcp.load(ref, storage_reader=FileSystemReader(str(dcp_checkpoint)))  # (also sets up any collectives outside the window)
    got = {k: torch.zeros_like(v) for k, v in like.items()}
    CachedMetadataFileSystemReader.clear_metadata_cache()
    reader = CachedMetadataFileSystemReader(str(dcp_checkpoint), load_on_engine=True, verify=verify)
    hold(eng._side.handle, cycles_per_ms)
    save(ckpt, sd, shm_dir / "a.pt")
    want = clone(sd)
    mutate(sd)
    seen = spy_entry(monkeypatch, eng, "load_boxes", queued_after(eng._side.handle))
    dcp.load(got, storage_reader=reader)
    assert seen == [False], "the window was closed (or the engine path was not taken)"
    stats = eng.last_box_load
    if staging_mb:
        assert stats["batches"] >= 4, stats
    if verify:
        assert stats["verified_records"] == len(like) and stats["unverified_records"] == 0, stats
    assert_same(got, ref, "dcp.load on the engine vs the stock reader")
    ckpt.finalize_async_save(blocking=True)
    assert_file(shm_dir / "a.pt", want)


# ---------------------------------------------------------------------------------------------------------------------
# 5. GPU checksums: _aux held
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("then", ["save", "restore"])
def test_gpu_crc_then(engines, ckpts, shm_dir, cycles_per_ms, monkeypatch, then):
    """Staging is free for the next writer only once the checksum kernel on _aux has read it, too."""
    monkeypatch.setenv("NVRX_B200_GPU_CRC", "1")
    monkeypatch.setenv("NVRX_B200_ZIP_CRC", "0")  # the record CRCs in the files can only come from the GPU
    eng, ckpt = engines(), ckpts()
    sd = make_state(6)
    reserve(eng, sd)
    assert eng._aux is not None  # created by the warm-up save: it can be held
    other = {k: v.cpu() for k, v in make_state(60).items()}
    hold(eng._aux.handle, cycles_per_ms)
    a = save(ckpt, sd, shm_dir / "a.pt")
    assert a.crc_info is not None
    want_a = clone(sd)
    mutate(sd)
    assert_open(queued_after(eng._aux.handle))  # the checksum kernel of a has not run yet
    if then == "save":
        save(ckpt, sd, shm_dir / "b.pt")
        want_b = clone(sd)
        mutate(sd)
    else:
        back = eng.restore(list(other.values()))
        assert_same(dict(zip(other, back)), other, "restored")
    ckpt.finalize_async_save(blocking=True)
    assert_file(shm_dir / "a.pt", want_a, crc_checked=True)
    if then == "save":
        assert_file(shm_dir / "b.pt", want_b, crc_checked=True)


# ---------------------------------------------------------------------------------------------------------------------
# 6. staging growth under a held drain
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("then", ["restore", "save"])
def test_staging_growth_under_held_drain(engines, ckpts, shm_dir, cycles_per_ms, then):
    """A 0.5 GB operation after a 150 MB save re-allocates staging: the old buffer may go only after its drain."""
    eng, ckpt = engines(), ckpts()
    small = make_state(7, n_big=2, big=(2048, 8192))
    reserve(eng, small)
    before = eng._staging.nbytes
    big = make_state(70)
    other = {k: v.cpu() for k, v in big.items()}
    hold(eng._side.handle, cycles_per_ms)
    a = save(ckpt, small, shm_dir / "a.pt")
    want_a = clone(small)
    mutate(small)
    assert not a.drained(), "the window was closed"
    if then == "restore":
        back = eng.restore(list(other.values()))
        assert_same(dict(zip(other, back)), other, "restored")
    else:
        save(ckpt, big, shm_dir / "b.pt")
        want_b = clone(big)
        mutate(big)
    assert eng._staging.nbytes > before
    ckpt.finalize_async_save(blocking=True)
    assert_file(shm_dir / "a.pt", want_a)
    if then == "save":
        assert_file(shm_dir / "b.pt", want_b)


# ---------------------------------------------------------------------------------------------------------------------
# 7. a released slot is reused while its drain is held
# ---------------------------------------------------------------------------------------------------------------------
def _abort_pending_save(how, eng, ckpt, sd, shm_dir):
    """Start a save with the drain held and abort it the way in-process restart does; returns the slot it had."""
    from nvidia_resiliency_ext.checkpointing.async_ckpt.core import AsyncCallsQueue, abort_nvrx_checkpoint
    from nvidia_resiliency_ext.checkpointing.local.basic_state_dict import BasicTensorAwareStateDict
    from nvidia_resiliency_ext.checkpointing.local.ckpt_managers.local_manager import LocalCheckpointManager

    if how == "manager":
        mgr, q = LocalCheckpointManager(shm_dir / "local"), AsyncCallsQueue(persistent=False)
        q.schedule_async_request(mgr.save(BasicTensorAwareStateDict(sd), 1, is_async=True))
    else:
        save(ckpt, sd, shm_dir / "a.pt")
    busy = [s for s in eng._slots if s.busy]
    assert len(busy) == 1
    abort_nvrx_checkpoint()
    if how == "manager":
        mgr.release_unfinalized()
    else:
        ckpt.finalize_async_save()  # the aborted call can never finalize: its slot goes back
    assert not busy[0].busy
    return busy[0]


@pytest.mark.parametrize("fill", ["gather", "readv_crc"])
@pytest.mark.parametrize("how", ["manager", "torch_ckpt"])
def test_released_slot_reused_by_restore(engines, ckpts, shm_dir, cycles_per_ms, dist_1rank, how, fill):
    """A restore that takes the slot of an aborted save fills it on the host; the aborted drain must not land on top."""
    from nvidia_resiliency_ext.checkpointing.b200 import ptzip
    from nvidia_resiliency_ext.checkpointing.b200.engine import choose_slot

    eng, ckpt = engines(), ckpts()
    sd = make_state(8)
    need = reserve(eng, sd)
    other = {k: v.cpu() for k, v in make_state(80).items()}
    kwargs = {}
    if fill == "readv_crc":
        torch.save(other, shm_dir / "other.pt")
        host = list(torch.load(shm_dir / "other.pt", mmap=True, weights_only=True).values())
        offs, crcs = ptzip.tensor_offsets_in_file(shm_dir / "other.pt", host), ptzip.record_crcs(shm_dir / "other.pt", len(host))
        assert offs is not None and crcs is not None and all(crcs)
        kwargs = {"file_source": (str(shm_dir / "other.pt"), offs), "expect_crcs": crcs}
    else:
        host = list(other.values())
    hold(eng._side.handle, cycles_per_ms)
    slot = _abort_pending_save(how, eng, ckpt, sd, shm_dir)
    mark = queued_after(eng._side.handle)
    assert choose_slot(eng._slots, need, eng.max_host_slots)[0] is slot  # the restore will fill the aborted save's slot
    assert_open(mark)
    back = eng.restore(host, **kwargs)
    assert_same(dict(zip(other, back)), other, "restored")


def test_released_slot_recreated_by_restore(engines, ckpts, shm_dir, cycles_per_ms):
    """A restore larger than the aborted save's slot re-creates that slot: its buffer may be unmapped only after the drain."""
    from nvidia_resiliency_ext.checkpointing.b200.engine import choose_slot

    eng, ckpt = engines(), ckpts()
    sd = make_state(9)
    reserve(eng, sd)
    other = {k: v.cpu() for k, v in make_state(90).items()}
    other["more"] = torch.randn(64 * MiB // 4)
    hold(eng._side.handle, cycles_per_ms)
    slot = _abort_pending_save("torch_ckpt", eng, ckpt, sd, shm_dir)
    mark = queued_after(eng._side.handle)
    old = slot.buf
    assert choose_slot(eng._slots, nbytes(other), eng.max_host_slots)[0] is slot and old.capacity < nbytes(other)
    assert_open(mark)
    back = eng.restore(list(other.values()))
    assert slot.buf is not old
    assert_same(dict(zip(other, back)), other, "restored")


# ---------------------------------------------------------------------------------------------------------------------
# 8. the progress word follows the bytes
# ---------------------------------------------------------------------------------------------------------------------
def test_progress_word_follows_the_bytes(engines, cycles_per_ms):
    """What a CPU-only writer relies on (open_snapshot_views): once the progress word says p, every byte below p is in the
    slot.  A thread polls the word through a held, multi-chunk drain and checks the 4 KiB below every new value."""
    eng = engines()
    sd = make_state(10)
    tensors = list(sd.values())
    reserve(eng, sd)
    want = [_bytes(t) for t in tensors]
    hold(eng._side.handle, cycles_per_ms)
    snap = eng.snapshot(tensors)
    mutate(sd)
    layout, hb = snap.layout, snap.slot.buf
    base = snap.progress_target - layout.total_bytes
    slot_bytes = hb.as_tensor(layout.total_bytes)
    segments = list(zip(layout.offsets, layout.packed_nbytes, want))
    seen, bad, first = [], [], []

    def poll():
        first.append(hb.progress)
        last, deadline = None, time.monotonic() + 30
        while time.monotonic() < deadline:
            p = hb.progress
            if p == last:
                continue
            last, q = p, p - base
            lo = max(0, q - 4096)
            for off, nb, ref in segments:
                a, b = max(lo, off), min(q, off + nb)
                if a < b and not torch.equal(slot_bytes[a:b], ref[a - off:b - off]):
                    bad.append((q, a, b))
            if 0 < q < layout.total_bytes:
                seen.append(q)
            if p == snap.progress_target:
                return

    th = threading.Thread(target=poll)
    th.start()
    assert not snap.drained(), "the window was closed"
    snap.wait()
    th.join()
    assert first == [base], "the poller started after the drain"
    assert not bad, f"progress ran ahead of the bytes: {bad[:5]}"
    assert len(set(seen)) >= 3, seen
    assert_same(dict(zip(sd, snap.host_views())), {k: w.view(t.dtype).reshape(t.shape) for (k, t), w in zip(sd.items(), want)}, "slot")
    snap.release()
