"""The engine's Python -- snapshot, restore, zero-copy publish / resident restore, GPU checksums, restore verification, the
TorchAsyncCheckpoint and LocalCheckpointManager GPU branches, the DCP writer's CUDA branch -- executed on the CPU against a
stand-in for the device at the C-ABI boundary (tests/_fake_device.py).  Not a parity test (the kernels are not involved): it
exists because that code was changed after the round's GPU budget was spent."""
import os
import zipfile
import zlib

import pytest
import torch

from _fake_device import FakeCudaTensor, fake_device, plain


def _state(seed=0, wrap=True):
    g = torch.Generator().manual_seed(seed)
    w = FakeCudaTensor.wrap if wrap else (lambda t: t)
    return {
        "model": {"w": w(torch.randn(700, 33, generator=g)), "ids": w(torch.arange(11) + seed), "empty": w(torch.empty(0, 3))},
        "opt": [w(torch.tensor(2.5 + seed)), {"m": w(torch.randn(4097, generator=g).to(torch.bfloat16))}],
        "blob": w(torch.randint(0, 255, (300_001,), dtype=torch.uint8, generator=g)),
        "iteration": 12345 + seed,
    }


def _flat(sd):
    from oracle import snapshot_oracle as orc

    return orc.flatten_tensors(sd)


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


def test_snapshot_and_restore_default_path(monkeypatch, built_library):
    with fake_device(monkeypatch) as (engine, lib):
        tensors = _flat(_state())
        snap = engine.snapshot(tensors)
        snap.wait()
        views = snap.host_views()
        assert len(views) == len(tensors) and all(not v.is_cuda for v in views)
        _same(views, tensors)
        assert snap.slot.buf.progress == snap.progress_target and snap.crc_info is None
        out = [FakeCudaTensor.wrap(torch.zeros_like(plain(t))) for t in tensors]
        back = engine.restore([v.clone() for v in views], out=out)
        _same(back, tensors)
        snap.release()
        assert lib.calls.count("pack") == 1 and lib.calls.count("scatter") == 1 and "fill" in lib.calls
        # narrow on save, widen on restore
        snap = engine.snapshot(tensors, narrow=True)
        host = snap.host_views()
        assert host[0].dtype == torch.bfloat16 and torch.equal(host[0], plain(tensors[0]).to(torch.bfloat16))
        widened = engine.restore(host, widen_to=[torch.float32 if t.dtype == torch.float32 else None for t in map(plain, tensors)],
                                 out=[FakeCudaTensor.wrap(torch.zeros_like(plain(t))) for t in tensors])
        assert torch.equal(plain(widened[0]), plain(tensors[0]).to(torch.bfloat16).to(torch.float32))
        snap.release()


@pytest.mark.parametrize("persistent", [True, False])
@pytest.mark.parametrize("gpu_crc", ["0", "1"])
def test_torch_async_checkpoint_zero_copy(monkeypatch, built_library, shm_dir, dist_1rank, persistent, gpu_crc):
    from nvidia_resiliency_ext.checkpointing.async_ckpt.torch_ckpt import TorchAsyncCheckpoint

    monkeypatch.setenv("NVRX_B200_ZERO_COPY", "1")
    monkeypatch.setenv("NVRX_B200_GPU_CRC", gpu_crc)
    with fake_device(monkeypatch) as (engine, lib):
        ckpt = TorchAsyncCheckpoint(persistent_queue=persistent)
        try:
            paths = [shm_dir / f"it{i}.pt" for i in range(4)]
            for i, path in enumerate(paths):
                sd = _state(i)
                want = _state(i, wrap=False)
                ckpt.async_save(sd, path)
                for t in _flat(sd):
                    if t.numel():
                        plain(t).zero_()  # training goes on
                ckpt.finalize_async_save(blocking=True)
                assert os.stat(path).st_nlink == 2, "hard link to the slot expected"
                _same(torch.load(path, weights_only=False), want)
                # record checksums are valid whoever computed them: the GPU kernel (opt-in) or the writer's threads (default)
                with zipfile.ZipFile(path) as zf:
                    for n in zf.namelist():
                        if not n.endswith("/.pad"):
                            zf.read(n)  # CRC check
                    assert zf.getinfo("archive/data/0").CRC == zlib.crc32(want["model"]["w"].numpy().tobytes())
                if i >= 1:
                    _same(torch.load(paths[i - 1], weights_only=False), _state(i - 1, wrap=False))  # not overwritten
                    os.unlink(paths[i - 1])
            assert len([s for s in engine._slots if s.buf is not None]) <= 3
            assert ("crc" in lib.calls) == (gpu_crc == "1")
        finally:
            ckpt.close()


def test_local_manager_zero_copy_resident_restore_and_verification(monkeypatch, built_library, shm_dir, dist_1rank):
    from nvidia_resiliency_ext.checkpointing.async_ckpt.core import AsyncCallsQueue
    from nvidia_resiliency_ext.checkpointing.b200._cabi import SnapError
    from nvidia_resiliency_ext.checkpointing.local.basic_state_dict import BasicTensorAwareStateDict
    from nvidia_resiliency_ext.checkpointing.local.ckpt_managers.local_manager import LocalCheckpointManager

    monkeypatch.setenv("NVRX_B200_ZERO_COPY", "1")
    monkeypatch.setenv("NVRX_B200_GPU_CRC", "1")
    monkeypatch.setenv("NVRX_B200_VERIFY_RESTORE", "1")
    with fake_device(monkeypatch) as (engine, lib):
        mgr = LocalCheckpointManager(shm_dir)
        q = AsyncCallsQueue(persistent=False)
        try:
            for it in (1, 2, 3):
                tasd = BasicTensorAwareStateDict(_state(10 + it))
                req = mgr.save(tasd, it, is_async=True)
                q.schedule_async_request(req)
                q.maybe_finalize_async_calls(blocking=True, no_dist=False)
                path = mgr._local_ckpt_path_from_id(mgr._ckpt_id(it))
                assert os.stat(path).st_nlink == 2
                assert mgr.find_latest() == it
                before = engine.resident_restores
                loaded, _ = mgr.load()
                assert engine.resident_restores == before + 1  # H2D fed from the pinned slot itself
                _same(loaded.state_dict, _state(10 + it, wrap=False))
            # a bit flips in the newest checkpoint: the verified restore refuses it
            reader = torch._C.PyTorchFileReader(str(path))
            off = reader.get_record_offset("data/0") + 1000
            del reader
            with open(path, "r+b") as fh:
                fh.seek(off)
                b = fh.read(1)
                fh.seek(off)
                fh.write(bytes([b[0] ^ 4]))
            mgr2 = LocalCheckpointManager(shm_dir)
            assert mgr2.find_latest() == 3
            with pytest.raises(SnapError, match="crc32 mismatch"):
                mgr2.load()
        finally:
            q.close()


def test_pread_restore(monkeypatch, built_library, tmp_path, dist_1rank):
    from nvidia_resiliency_ext.checkpointing.local.basic_state_dict import BasicTensorAwareStateDict
    from nvidia_resiliency_ext.checkpointing.local.ckpt_managers.local_manager import LocalCheckpointManager

    monkeypatch.setenv("NVRX_B200_RESTORE_PREAD", "1")
    with fake_device(monkeypatch) as (engine, lib):
        mgr = LocalCheckpointManager(tmp_path)
        mgr.save(BasicTensorAwareStateDict(_state(5)), 9, is_async=False)
        assert mgr.find_latest() == 9
        gathers = []
        from nvidia_resiliency_ext.checkpointing.b200.engine import HostBuffer

        monkeypatch.setattr(HostBuffer, "gather", lambda self, *a, **k: gathers.append(1))
        loaded, _ = mgr.load()
        assert not gathers and engine.file_restores == 1  # file -> pinned ring -> staging (nvrx_fill_from_fd), no slot, no mmap gather
        assert "fill_from_fd" in lib.calls and not any(s.busy for s in engine._slots)
        _same(loaded.state_dict, _state(5, wrap=False))
        # opt-out: the mmap gather into a pinned slot
        monkeypatch.setenv("NVRX_B200_RESTORE_PREAD", "0")
        mgr2 = LocalCheckpointManager(tmp_path)
        assert mgr2.find_latest() == 9
        loaded, _ = mgr2.load()
        assert gathers and engine.file_restores == 1


def test_dcp_writer_cuda_branch(monkeypatch, built_library, tmp_path, dist_1rank):
    import filecmp

    import torch.distributed.checkpoint as dcp
    from torch.distributed.checkpoint import DefaultSavePlanner, FileSystemReader, FileSystemWriter

    from nvidia_resiliency_ext.checkpointing.async_ckpt.core import AsyncCallsQueue, AsyncRequest
    from nvidia_resiliency_ext.checkpointing.async_ckpt.filesystem_async import FileSystemWriterAsync
    from nvidia_resiliency_ext.checkpointing.async_ckpt.state_dict_saver import save_state_dict_async_finalize, save_state_dict_async_plan

    with fake_device(monkeypatch) as (engine, lib):
        host_state = {"model": {"w": torch.randn(33, 17), "h": torch.randn(5, 3).to(torch.bfloat16)}, "opt": {"step": torch.tensor(3), "lr": 0.5}}
        dev_state = {"model": {k: FakeCudaTensor.wrap(v.clone()) for k, v in host_state["model"].items()}, "opt": dict(host_state["opt"])}
        dcp.save(host_state, storage_writer=FileSystemWriter(tmp_path / "sync", thread_count=2), planner=DefaultSavePlanner())
        q = AsyncCallsQueue(persistent=True)
        try:
            writer = FileSystemWriterAsync(tmp_path / "async", thread_count=2)
            ret = save_state_dict_async_plan(dev_state, writer, None, 0, planner=DefaultSavePlanner())
            assert writer._snapshot is not None and len(writer._payload["cuda_indices"]) == 2
            save_fn, preload_fn, save_args = writer.get_save_function_and_args()
            q.schedule_async_request(AsyncRequest(save_fn, save_args, [lambda: save_state_dict_async_finalize(*ret)], preload_fn=preload_fn))
            for v in dev_state["model"].values():
                plain(v).zero_()
            q.maybe_finalize_async_calls(blocking=True)
            assert writer._snapshot is None
        finally:
            q.close()
        names = sorted(f for f in os.listdir(tmp_path / "sync") if f.endswith(".distcp"))
        _, mismatch, errors = filecmp.cmpfiles(tmp_path / "sync", tmp_path / "async", names, shallow=False)
        assert names and not mismatch and not errors
        got = {"model": {k: torch.zeros_like(v) for k, v in host_state["model"].items()}, "opt": {"step": torch.tensor(0), "lr": None}}
        dcp.load(got, storage_reader=FileSystemReader(tmp_path / "async"))
        assert torch.equal(got["model"]["w"], host_state["model"]["w"]) and got["opt"]["lr"] == 0.5


@pytest.mark.parametrize("persistent", [True, False])
def test_default_paths_torch_async_and_local_manager(monkeypatch, built_library, shm_dir, tmp_path, dist_1rank, persistent):
    """NVRX_B200_ZERO_COPY=0 (the default is the hard-link publish): the copying writer, slot release on finalize, cleanup of
    older iterations, restore from the file."""
    from nvidia_resiliency_ext.checkpointing.async_ckpt.core import AsyncCallsQueue
    from nvidia_resiliency_ext.checkpointing.async_ckpt.torch_ckpt import TorchAsyncCheckpoint
    from nvidia_resiliency_ext.checkpointing.local.basic_state_dict import BasicTensorAwareStateDict
    from nvidia_resiliency_ext.checkpointing.local.ckpt_managers.local_manager import LocalCheckpointManager
    from nvidia_resiliency_ext.checkpointing.utils import preload_tensors

    for var in ("NVRX_B200_GPU_CRC", "NVRX_B200_VERIFY_RESTORE", "NVRX_B200_RESTORE_PREAD"):
        monkeypatch.delenv(var, raising=False)
    from nvidia_resiliency_ext.checkpointing.b200 import fastsave

    monkeypatch.delenv("NVRX_B200_ZERO_COPY", raising=False)
    assert fastsave.zero_copy_enabled() and not fastsave.replicated_zero_copy_enabled()  # the defaults
    monkeypatch.setenv("NVRX_B200_ZERO_COPY", "0")
    with fake_device(monkeypatch) as (engine, lib):
        ckpt = TorchAsyncCheckpoint(persistent_queue=persistent)
        try:
            for i in range(3):
                path = shm_dir / f"plain{i}.pt"
                ckpt.async_save(_state(i), path)
                ckpt.finalize_async_save(blocking=True)
                assert os.stat(path).st_nlink == 1  # a copy, not a link
                _same(torch.load(path, weights_only=False), _state(i, wrap=False))
                with zipfile.ZipFile(path) as z:  # default mode: every record carries its checksum, like a torch.save file
                    assert z.testzip() is None and all(zi.CRC for zi in z.infolist() if "/data/" in zi.filename and zi.file_size)
            assert len(engine._slots) == 2 and not any(s.busy for s in engine._slots)
        finally:
            ckpt.close()
        host, snap = preload_tensors(_state(7), non_blocking=True, return_snapshot=True)
        snap.wait()
        _same(host, _state(7, wrap=False))
        snap.release()

        mgr = LocalCheckpointManager(tmp_path / "ckpt")
        q = AsyncCallsQueue(persistent=False)
        try:
            for it in (1, 2):
                req = mgr.save(BasicTensorAwareStateDict(_state(20 + it)), it, is_async=True)
                q.schedule_async_request(req)
                q.maybe_finalize_async_calls(blocking=True, no_dist=False)
            import time

            time.sleep(0.5)  # cleanup of iteration 1 runs in a background thread
            assert sorted(p.name for p in mgr.local_ckpt_dir.iterdir()) == ["iter_0000002_0_local.pt"]
            with zipfile.ZipFile(mgr.local_ckpt_dir / "iter_0000002_0_local.pt") as z:
                assert z.testzip() is None
            assert mgr.find_latest() == 2
            loaded, _ = mgr.load()
            _same(loaded.state_dict, _state(22, wrap=False))
            assert all(t.is_cuda for t in loaded.tensors) and engine.resident_restores == 0
        finally:
            q.close()


def test_abort_gives_host_slots_back(monkeypatch, built_library, shm_dir, dist_1rank):
    """In-process restart: aborted saves never finalize; their pinned slots must come back or the pool runs dry."""
    from nvidia_resiliency_ext.checkpointing.async_ckpt.core import AsyncCallsQueue, AsyncRequest, abort_nvrx_checkpoint
    from nvidia_resiliency_ext.checkpointing.async_ckpt.filesystem_async import FileSystemWriterAsync
    from nvidia_resiliency_ext.checkpointing.async_ckpt.state_dict_saver import save_state_dict_async_plan
    from nvidia_resiliency_ext.checkpointing.async_ckpt.torch_ckpt import TorchAsyncCheckpoint

    with fake_device(monkeypatch) as (engine, lib):
        ckpt = TorchAsyncCheckpoint(persistent_queue=True)
        q = AsyncCallsQueue(persistent=True)
        try:
            # two saves in flight (they hold two of the four slots of the pool), then the abort
            ckpt.async_save(_state(0), shm_dir / "a0.pt")
            dev_state = {"m": {"w": FakeCudaTensor.wrap(torch.randn(100, 10))}}
            writer = FileSystemWriterAsync(shm_dir / "dcp0", thread_count=1)
            save_state_dict_async_plan(dev_state, writer, None, 0)
            save_fn, preload_fn, save_args = writer.get_save_function_and_args()
            q.schedule_async_request(AsyncRequest(save_fn, save_args, [], preload_fn=preload_fn))
            abort_nvrx_checkpoint()
            del writer  # the aborted DCP save never reaches retrieve_write_results
            for i in range(5):  # more saves than the pool has slots: they only fit if the aborted ones gave theirs back
                ckpt.async_save(_state(100 + i), shm_dir / f"b{i}.pt")
                if i % 2:
                    ckpt.finalize_async_save(blocking=True)
            ckpt.finalize_async_save(blocking=True)
            _same(torch.load(shm_dir / "b4.pt", weights_only=False), _state(104, wrap=False))
            assert len(engine._slots) <= engine.max_host_slots and not any(s.busy for s in engine._slots)
        finally:
            ckpt.close()
            q.close()


def test_warmup_creates_the_resources_of_the_first_save(monkeypatch, built_library, shm_dir, dist_1rank):
    from nvidia_resiliency_ext.checkpointing.async_ckpt.torch_ckpt import TorchAsyncCheckpoint

    with fake_device(monkeypatch) as (engine, lib):
        ckpt = TorchAsyncCheckpoint(persistent_queue=False)
        try:
            sd = _state(3)
            nbytes = ckpt.warmup(sd)
            assert nbytes > 0 and engine._staging is not None and engine._staging.nbytes >= nbytes
            bufs = [s.buf.name for s in engine._slots]
            assert all(s.buf is not None and s.buf.capacity >= nbytes and not s.busy for s in engine._slots)
            plans = len(engine._plans)
            ckpt.async_save(sd, shm_dir / "w.pt")
            ckpt.finalize_async_save(blocking=True)
            assert [s.buf.name for s in engine._slots] == bufs and len(engine._plans) == plans  # nothing new was allocated
            _same(torch.load(shm_dir / "w.pt", weights_only=False), _state(3, wrap=False))
            assert ckpt.warmup({"x": torch.ones(3)}) == 0  # host state: nothing to prepare
        finally:
            ckpt.close()


def test_reserve_sizes_slots_for_a_zero_copy_save(monkeypatch, built_library, shm_dir, dist_1rank):
    """reserve(packed bytes, tensors) leaves room for the checkpoint file's records and directory behind the payload: the
    zero-copy save of that size that follows allocates and pins no new host buffer inside the call."""
    from nvidia_resiliency_ext.checkpointing.async_ckpt.torch_ckpt import TorchAsyncCheckpoint

    monkeypatch.setenv("NVRX_B200_ZERO_COPY", "1")
    with fake_device(monkeypatch) as (engine, lib):
        ckpt = TorchAsyncCheckpoint(persistent_queue=False)
        try:
            sd = _state(5)
            tensors = _flat(sd)
            engine.reserve(sum(t.numel() * t.element_size() for t in tensors) + (1 << 20), len(tensors))
            bufs = [s.buf.name for s in engine._slots if s.buf is not None]
            assert bufs
            ckpt.async_save(sd, shm_dir / "r.pt")
            ckpt.finalize_async_save(blocking=True)
            assert [s.buf.name for s in engine._slots if s.buf is not None] == bufs
            assert os.stat(shm_dir / "r.pt").st_nlink > 1  # published by the hard link, not copied
            _same(torch.load(shm_dir / "r.pt", weights_only=False), _state(5, wrap=False))
        finally:
            ckpt.close()


@pytest.mark.parametrize("seed,persistent", [(1, False), (2, False), (3, False), (4, True)])
def test_random_sequences_of_saves_deletes_restores(monkeypatch, built_library, shm_dir, tmp_path, dist_1rank, seed, persistent):
    """Slot life cycle under a random workload: zero-copy and copying saves to /dev/shm and to another file system, files
    deleted or kept, structures changing, trims in between.  Invariants: every file that exists loads back exactly, kept files
    are never disturbed by later snapshots, the pool respects its bound, nothing stays busy."""
    import random

    from nvidia_resiliency_ext.checkpointing.async_ckpt.torch_ckpt import TorchAsyncCheckpoint

    rng = random.Random(seed)
    monkeypatch.setenv("NVRX_B200_GPU_CRC", "1" if seed == 2 else "0")
    with fake_device(monkeypatch) as (engine, lib):
        ckpt = TorchAsyncCheckpoint(persistent_queue=persistent)  # the persistent worker keeps slot mappings cached
        alive = {}  # path -> expected state
        try:
            for step in range(14):
                monkeypatch.setenv("NVRX_B200_ZERO_COPY", rng.choice(["1", "1", "0"]))
                base = shm_dir if rng.random() < 0.75 else tmp_path
                path = base / f"s{step}.pt"
                sd = _state(step)
                if rng.random() < 0.3:  # a structure change: other sizes, one tensor more
                    sd["model"]["extra"] = FakeCudaTensor.wrap(torch.randn(rng.randint(1, 5000)))
                want = {"model": {k: plain(v).clone() for k, v in sd["model"].items()}, "opt": [plain(sd["opt"][0]).clone(), {"m": plain(sd["opt"][1]["m"]).clone()}],
                        "blob": plain(sd["blob"]).clone(), "iteration": sd["iteration"]}
                ckpt.async_save(sd, path)
                for t in _flat(sd):
                    if t.numel():
                        plain(t).zero_()
                ckpt.finalize_async_save(blocking=True)
                alive[path] = want
                for p, w in alive.items():  # nothing that is still on disk was disturbed
                    _same(torch.load(p, weights_only=False), w)
                if rng.random() < 0.6 and len(alive) > 1:
                    victim = rng.choice(list(alive)[:-1])
                    os.unlink(victim)
                    del alive[victim]
                if rng.random() < 0.15:
                    engine.trim()
                assert len(engine._slots) <= engine.max_host_slots and not any(s.busy for s in engine._slots)
            assert len(engine._plans) <= 2 * 14 + 2
        finally:
            ckpt.close()


def test_local_manager_gives_slots_back_after_abort(monkeypatch, built_library, shm_dir, tmp_path, dist_1rank):
    """ADVICE r1: aborted LocalCheckpointManager saves never run their finalize_fn; without reaping, four of them pin the
    whole slot pool and every later save fails with 'all 4 slots hold unfinalized snapshots'."""
    from nvidia_resiliency_ext.checkpointing.async_ckpt.core import AsyncCallsQueue, abort_nvrx_checkpoint
    from nvidia_resiliency_ext.checkpointing.local.basic_state_dict import BasicTensorAwareStateDict
    from nvidia_resiliency_ext.checkpointing.local.ckpt_managers.local_manager import LocalCheckpointManager

    with fake_device(monkeypatch) as (engine, lib):
        mgr = LocalCheckpointManager(tmp_path / "ckpt")
        q = AsyncCallsQueue(persistent=False)
        try:
            for it in range(1, 8):  # more aborted saves than the pool has slots
                req = mgr.save(BasicTensorAwareStateDict(_state(it)), it, is_async=True)
                q.schedule_async_request(req)
                abort_nvrx_checkpoint()  # in-process restart: the queue forgets the call, finalize_fn never runs
                for p in mgr.local_ckpt_dir.glob("iter_*"):
                    p.unlink()  # whatever the killed child left behind
            req = mgr.save(BasicTensorAwareStateDict(_state(50)), 50, is_async=True)
            q.schedule_async_request(req)
            q.maybe_finalize_async_calls(blocking=True, no_dist=False)
            assert mgr.find_latest() == 50
            busy = [s for s in engine._slots if s.busy]
            assert len(busy) <= 1, "only the stale request still referenced by `req` bookkeeping may hold a slot"
            mgr.release_unfinalized()
            assert not any(s.busy for s in engine._slots)
            # a request that was handed out but not scheduled yet keeps its slot while the caller holds it ...
            pending = mgr.save(BasicTensorAwareStateDict(_state(60)), 60, is_async=True)
            mgr._reap_abandoned()
            assert sum(s.busy for s in engine._slots) == 1
            pending.execute_sync()  # ... and can still be executed (the reference tests drive saves this way)
            assert not any(s.busy for s in engine._slots) and mgr.find_latest() == 60
            # a synchronous save that fails releases its slot as well
            monkeypatch.setattr(mgr, "_save", lambda *a, **k: (_ for _ in ()).throw(OSError("disk full")))
            with pytest.raises(OSError):
                mgr.save(BasicTensorAwareStateDict(_state(70)), 70, is_async=False)
            assert not any(s.busy for s in engine._slots)
        finally:
            q.close()


def test_async_save_of_a_dict_with_host_tensors(monkeypatch, built_library, shm_dir, dist_1rank):
    """ADVICE r1: {'model': cuda tensors, 'rng_state': torch.get_rng_state()} is a common training state dict; the reference's
    preload_tensors passes host tensors through, so must async_save."""
    from nvidia_resiliency_ext.checkpointing.async_ckpt.torch_ckpt import TorchAsyncCheckpoint

    for persistent in (False, True):
        with fake_device(monkeypatch) as (engine, lib):
            ckpt = TorchAsyncCheckpoint(persistent_queue=persistent)
            try:
                sd = _state(5)
                want = _state(5, wrap=False)
                rng = torch.get_rng_state()
                sd["rng_state"], want["rng_state"] = rng, rng.clone()
                sd["extra"] = {"cpu_list": [torch.arange(7), 3.5, "text"]}
                want["extra"] = {"cpu_list": [torch.arange(7), 3.5, "text"]}
                path = shm_dir / f"mixed{int(persistent)}.pt"
                ckpt.async_save(sd, path)
                ckpt.finalize_async_save(blocking=True)
                with zipfile.ZipFile(path) as z:
                    assert z.testzip() is None  # slot records and the pass-through host tensors alike
                got = torch.load(path, weights_only=False)
                assert torch.equal(got["rng_state"], want["rng_state"]) and got["extra"]["cpu_list"][1:] == [3.5, "text"]
                assert torch.equal(got["extra"]["cpu_list"][0], torch.arange(7))
                got.pop("rng_state"), got.pop("extra"), want.pop("rng_state"), want.pop("extra")
                _same(got, want)
            finally:
                ckpt.close()


def _mcore_like(seed, fake=True):
    from _mcore_like import MCoreLikeTensorAwareStateDict

    g = torch.Generator().manual_seed(seed)
    wrap = FakeCudaTensor.wrap if fake else (lambda t: t)
    model = {f"layers.{i}.w": wrap(torch.randn(33 + i, 17, generator=g)) for i in range(3)}
    optim = {i: {"exp_avg": wrap(torch.randn(33 + i, 17, generator=g)), "step": wrap(torch.tensor(float(i)))} for i in range(3)}
    return MCoreLikeTensorAwareStateDict.from_state_dict(model, optim, iteration=seed)


def test_mcore_shaped_state_dict_goes_through_the_engine(monkeypatch, built_library, shm_dir, tmp_path, dist_1rank):
    """Row f4: a third-party TensorAwareStateDict with Megatron-Core's shape (tensors inside ShardedTensor-like objects, a
    `common` part, its own per-tensor copy methods) is snapshotted and restored by the engine through the ABC contract alone."""
    from nvidia_resiliency_ext.checkpointing.async_ckpt.core import AsyncCallsQueue
    from nvidia_resiliency_ext.checkpointing.local.ckpt_managers.local_manager import LocalCheckpointManager

    with fake_device(monkeypatch) as (engine, lib):
        mgr = LocalCheckpointManager(shm_dir / "mc")
        q = AsyncCallsQueue(persistent=False)
        try:
            tasd = _mcore_like(3)
            want = [plain(t).clone() for t in tasd.tensors]
            before = len(lib.calls)
            req = mgr.save(tasd, 5, is_async=True)
            assert "pack" in lib.calls[before:] and tasd.calls == []  # engine path, not the class's own per-tensor copies
            assert not tasd.is_hollow and all(not t.is_cuda for t in tasd.tensors)  # host views were inserted back
            q.schedule_async_request(req)
            q.maybe_finalize_async_calls(blocking=True, no_dist=False)
            assert not any(s.busy for s in engine._slots)
            mgr2 = LocalCheckpointManager(shm_dir / "mc")
            assert mgr2.find_latest() == 5
            loaded, cid = mgr2.load()
            assert loaded.calls == [] and engine.file_restores == 1  # restored by the engine from the file
            assert loaded.common["iteration"] == 3 and loaded.sharded_state_dict["rerun"].data == {"mode": "disabled"}
            got = list(loaded.tensors)
            assert len(got) == len(want) and all(t.is_cuda and torch.equal(plain(t), w) for t, w in zip(got, want))
            sh = loaded.sharded_state_dict["model"]["layers.1.w"]
            assert sh.key == "model.layers.1.w" and sh.global_offset == (0, 0) and sh.local_shape == (34, 17)
            # opt-out keeps the class's own methods (reference behaviour)
            monkeypatch.setenv("NVRX_B200_GENERIC_TASD", "0")
            monkeypatch.setattr(torch.cuda, "synchronize", lambda *a, **k: None)  # the reference path ends in a device sync
            tasd = _mcore_like(4)
            mgr.save(tasd, 6, is_async=False)
            assert tasd.calls == ["copy_tensors_to_cpu"]
        finally:
            q.close()


def test_preload_tensors_views_keep_their_slot_and_give_it_back(monkeypatch, built_library, dist_1rank):
    """ADVICE r1: preload_tensors() without return_snapshot hands out views of a pooled slot and no handle -- the slot must stay
    reserved while a view is alive and come back afterwards (it used to stay busy for good)."""
    import gc

    from nvidia_resiliency_ext.checkpointing.utils import preload_tensors

    with fake_device(monkeypatch) as (engine, lib):
        kept = []
        for i in range(6):  # more calls than the pool has slots
            host = preload_tensors(_state(i), non_blocking=False)
            _same(host, _state(i, wrap=False))
            busy = [s for s in engine._slots if s.busy]
            assert len(busy) == 1 + len(kept)
            if i == 0:
                kept.append(host)  # one result stays alive: its slot must not be handed out again
            del host
            gc.collect()
            assert sum(s.busy for s in engine._slots) == len(kept)
        _same(kept[0], _state(0, wrap=False))  # still intact after five more snapshots
        kept.clear()
        gc.collect()
        assert not any(s.busy for s in engine._slots)


@pytest.mark.parametrize("zero_copy", ["1", "0"])
def test_restoring_the_state_dict_that_was_just_saved(monkeypatch, built_library, tmp_path, dist_1rank, zero_copy):
    """Reference test_basic_local.py:62-64: after save() the caller's state dict holds host tensors -- here views of the
    snapshot slot, which is free again once the save is finalized -- and ``restore_tensor_device()`` on it must give the
    original values back.  With the container geometry of the default mode the views do not sit at the dense offsets of a
    restore plan; gathering them into "a free slot" picked the slot they live in."""
    from nvidia_resiliency_ext.checkpointing.local.basic_state_dict import BasicTensorAwareStateDict
    from nvidia_resiliency_ext.checkpointing.local.ckpt_managers.local_manager import LocalCheckpointManager

    monkeypatch.setenv("NVRX_B200_ZERO_COPY", zero_copy)
    with fake_device(monkeypatch) as (engine, lib):
        mgr = LocalCheckpointManager(tmp_path / "disk")  # not /dev/shm: the slot is released, not published
        sd = BasicTensorAwareStateDict(_state(8))
        mgr.save(sd, 1, is_async=False)
        assert not any(s.busy for s in engine._slots) and all(not t.is_cuda for t in sd.tensors)
        before = engine.resident_restores
        sd.restore_tensor_device()
        assert engine.resident_restores == before + 1 and not any(s.busy for s in engine._slots)
        _same(sd.state_dict, _state(8, wrap=False))
        # scrambled views of a slot (not ascending) are taken out of the slot before anything is gathered
        host = BasicTensorAwareStateDict(_state(9))
        snap = host.copy_tensors_to_cpu(non_blocking=False)
        views = list(host.tensors)[::-1]
        snap.release()
        back = engine.restore(views)
        want = _flat(_state(9, wrap=False))[::-1]
        assert all(torch.equal(plain(a), b) for a, b in zip(back, want))


from test_ptl_glue_cpu import glue  # noqa: E402,F401  (fixture: stub of the three lightning symbols the glue imports)


def test_ptl_glue_drives_the_local_manager(glue, monkeypatch, built_library, shm_dir, dist_1rank):  # noqa: F811
    """CPU twin of tests/test_gpu_zzy_ptl_glue.py::test_ptl_glue_drives_the_local_manager_on_gpu (same flow on the stand-in device)."""
    from nvidia_resiliency_ext.checkpointing.async_ckpt.core import AsyncCallsQueue
    from nvidia_resiliency_ext.checkpointing.local.basic_state_dict import BasicTensorAwareStateDict
    from nvidia_resiliency_ext.checkpointing.local.ckpt_managers.local_manager import LocalCheckpointManager

    class IO(glue.HierarchicalCheckpointIO):
        def to_tensor_aware_state_dict(self, checkpoint):
            return BasicTensorAwareStateDict(checkpoint)

        def from_tensor_aware_state_dict(self, tasd, **kw):
            return tasd.state_dict

    class GlobalIO:
        def load_checkpoint(self, path, map_location=None, **kw):
            return {"from": "global"}

        def save_checkpoint(self, *a, **k):
            raise AssertionError("a local save must not reach the global CheckpointIO")

    with fake_device(monkeypatch) as (engine, lib):
        mgr = LocalCheckpointManager(shm_dir / "ptl")
        io = IO(GlobalIO(), mgr, get_global_ckpt_iteration_fn=lambda p: int(str(p).rsplit("=", 1)[-1]), async_save=True)
        q = AsyncCallsQueue(persistent=False)
        g = torch.Generator().manual_seed(21)
        state = {f"param_{i}": FakeCudaTensor.wrap(torch.rand(513, 255, generator=g)) for i in range(6)}
        want = {k: plain(v).clone() for k, v in state.items()}

        class Trainer:
            global_step = 40

            def save_checkpoint(self, path, storage_options=None):
                req = io.save_checkpoint({"state_dict": dict(state), "global_step": self.global_step}, path, storage_options)
                q.schedule_async_request(req)

        try:
            cb = glue.LocalCheckpointCallback(every_n_train_steps=20)
            cb._save_last_checkpoint(Trainer(), {})
            q.maybe_finalize_async_calls(blocking=True, no_dist=False)
            assert io.load_checkpoint("/global/step=50") == {"from": "global"}
            io2 = IO(GlobalIO(), LocalCheckpointManager(shm_dir / "ptl"), get_global_ckpt_iteration_fn=lambda p: 30)
            resumed = io2.load_checkpoint("/global/step=30")
            assert resumed["global_step"] == 40
            assert all(resumed["state_dict"][k].is_cuda and torch.equal(plain(resumed["state_dict"][k]), w) for k, w in want.items())
        finally:
            q.close()


def test_restore_of_arbitrary_mixes_of_slot_views_and_host_tensors(monkeypatch, built_library, dist_1rank):
    """engine.restore must give every tensor back whatever mix it is handed: views of a slot in order (read in place), in any
    other order or only some of them (taken out of the slot first), views of two different slots, plain host tensors."""
    import random

    with fake_device(monkeypatch) as (engine, lib):
        rng = random.Random(7)
        for trial in range(25):
            a = [FakeCudaTensor.wrap(torch.randn(rng.choice([1, 7, 64, 513, 4097]), generator=torch.Generator().manual_seed(trial * 10 + i))) for i in range(rng.randint(1, 6))]
            b = [FakeCudaTensor.wrap(torch.randn(rng.choice([3, 100, 2048]), generator=torch.Generator().manual_seed(trial * 10 + 50 + i))) for i in range(rng.randint(1, 4))]
            sa, sb = engine.snapshot(a), engine.snapshot(b)
            sa.wait(), sb.wait()
            pool = [(v, plain(t).clone()) for v, t in zip(sa.host_views(), a)] + [(v, plain(t).clone()) for v, t in zip(sb.host_views(), b)]
            pool += [(torch.full((rng.randint(1, 300),), float(trial)), None)]
            mode = trial % 5
            if mode == 0:
                pick = pool[: len(a)]  # one slot, in order -> in place
            elif mode == 1:
                pick = list(reversed(pool[: len(a)]))
            elif mode == 2:
                pick = rng.sample(pool, rng.randint(1, len(pool)))
            elif mode == 3:
                pick = pool[len(a) : len(a) + len(b)] + pool[: len(a)]  # two slots
            else:
                pick = [pool[-1]] + pool[: len(a)]  # a plain host tensor in front of slot views
            if rng.random() < 0.5:
                sa.release(), sb.release()  # the slots may be handed out again by the restore itself
            got = engine.restore([v for v, _ in pick])
            for g, (v, want) in zip(got, pick):
                want = want if want is not None else v
                assert g.is_cuda and torch.equal(plain(g), plain(want)), (trial, mode)
            if not sa.released:
                sa.release(), sb.release()
            assert not any(s.busy for s in engine._slots)
