"""Zero-copy persistence on the GPU (the default since round 2; ``NVRX_B200_ZERO_COPY=0`` opts out): the pinned slot a snapshot drains into IS the
checkpoint file on /dev/shm (hard link), so a save is durable as soon as its drain has finished.

The host half is covered on the CPU (tests/test_zero_copy_cpu.py)."""
import os

import pytest
import torch

pytestmark = pytest.mark.gpu  # part of the default suite


def _state(seed, n=12):
    g = torch.Generator(device="cuda").manual_seed(seed)
    sd = {f"p{i}": torch.randn(1024, 257 + i, device="cuda", generator=g) for i in range(n)}
    sd["nested"] = {"ids": torch.randint(0, 100, (1000,), device="cuda", generator=g), "step": torch.tensor(3.0, device="cuda"), "tag": "x"}
    sd["half"] = torch.randn(333, device="cuda", generator=g).to(torch.bfloat16)
    return sd


def _equal(a, b):
    if isinstance(a, dict):
        return list(a) == list(b) and all(_equal(a[k], b[k]) for k in a)
    if isinstance(a, torch.Tensor):
        return a.dtype == b.dtype and torch.equal(a.cpu(), b.cpu())
    return a == b


@pytest.mark.parametrize("persistent", [True, False])
def test_torch_async_checkpoint_publishes_slots(shm_dir, dist_1rank, built_library, monkeypatch, persistent):
    from nvidia_resiliency_ext.checkpointing.async_ckpt.torch_ckpt import TorchAsyncCheckpoint
    from nvidia_resiliency_ext.checkpointing.b200.engine import SnapshotEngine

    monkeypatch.setenv("NVRX_B200_ZERO_COPY", "1")
    ckpt = TorchAsyncCheckpoint(persistent_queue=persistent)
    engine = SnapshotEngine.get()
    paths = [shm_dir / f"it{i}.pt" for i in range(4)]
    try:
        for i, path in enumerate(paths):
            sd = _state(i)
            ckpt.async_save(sd, path)
            for t in (v for v in sd.values() if isinstance(v, torch.Tensor)):
                t.zero_()  # training goes on
            ckpt.finalize_async_save(blocking=True)
            assert os.stat(path).st_nlink == 2, "the checkpoint must be a hard link to the slot, not a copy"
            # every checkpoint written so far is intact: no later snapshot went into a published slot
            for j in range(max(0, i - 1), i + 1):
                assert _equal(torch.load(paths[j], weights_only=False, map_location="cuda"), _state(j)), (i, j)
            if i >= 1:
                os.unlink(paths[i - 1])  # what a manager's cleanup does: frees that slot for the next save
        assert len([s for s in engine._slots if s.buf is not None]) <= 3
    finally:
        ckpt.close()


def test_local_manager_zero_copy_roundtrip(shm_dir, dist_1rank, built_library, monkeypatch):
    from nvidia_resiliency_ext.checkpointing.async_ckpt.core import AsyncCallsQueue
    from nvidia_resiliency_ext.checkpointing.local.basic_state_dict import BasicTensorAwareStateDict
    from nvidia_resiliency_ext.checkpointing.local.ckpt_managers.local_manager import LocalCheckpointManager

    from nvidia_resiliency_ext.checkpointing.b200.engine import SnapshotEngine

    monkeypatch.setenv("NVRX_B200_ZERO_COPY", "1")
    engine = SnapshotEngine.get()
    before = engine.resident_restores
    mgr = LocalCheckpointManager(shm_dir)
    q = AsyncCallsQueue(persistent=False)
    try:
        for it in (1, 2, 3):
            tasd = BasicTensorAwareStateDict(_state(100 + it))
            live = list(tasd.tensors)
            q.schedule_async_request(mgr.save(tasd, it, is_async=True))
            for t in live:
                t.zero_()
            q.maybe_finalize_async_calls(blocking=True, no_dist=False)
            path = mgr._local_ckpt_path_from_id(mgr._ckpt_id(it))
            assert os.stat(path).st_nlink == 2
            assert mgr.find_latest() == it
            loaded, _ = mgr.load()
            assert _equal(loaded.state_dict, _state(100 + it))
            assert all(t.is_cuda for t in loaded.tensors)
        # every load found its file to be a live pinned slot and fed the H2D from it (no host-side gather)
        assert engine.resident_restores == before + 3
    finally:
        q.close()


def test_restore_through_pread(tmp_path, shm_dir, dist_1rank, built_library, monkeypatch):
    """Default restore of a local checkpoint: parallel pread from the file (any file system) into the pinned ring, chunk-pipelined
    H2D (nvrx_fill_from_fd), one scatter kernel."""
    from nvidia_resiliency_ext.checkpointing.local.basic_state_dict import BasicTensorAwareStateDict
    from nvidia_resiliency_ext.checkpointing.local.ckpt_managers.local_manager import LocalCheckpointManager

    monkeypatch.setenv("NVRX_B200_RESTORE_PREAD", "1")
    for root in (tmp_path / "disk", shm_dir / "ram"):
        mgr = LocalCheckpointManager(root)
        mgr.save(BasicTensorAwareStateDict(_state(55)), 4, is_async=False)
        assert mgr.find_latest() == 4
        from nvidia_resiliency_ext.checkpointing.b200.engine import SnapshotEngine

        eng = SnapshotEngine.get()
        before = eng.file_restores + eng.resident_restores
        loaded, _ = mgr.load()
        assert _equal(loaded.state_dict, _state(55)) and all(t.is_cuda for t in loaded.tensors)
        # from the file through the ring, or -- on /dev/shm, where the file IS a still-pinned slot of this process -- in place
        assert eng.file_restores + eng.resident_restores == before + 1
        mgr_fresh = LocalCheckpointManager(root)
        os.environ["NVRX_B200_ZERO_COPY"] = "0"  # what a freshly started process sees: no resident slot, the file path
        try:
            assert mgr_fresh.find_latest() == 4
            files = eng.file_restores
            loaded, _ = mgr_fresh.load()
            assert _equal(loaded.state_dict, _state(55)) and eng.file_restores == files + 1
        finally:
            os.environ["NVRX_B200_ZERO_COPY"] = "1"
