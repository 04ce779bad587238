"""GPU test of torch.distributed.checkpoint loads on the engine (``CachedMetadataFileSystemReader(load_on_engine=True)``):
the loaded CUDA tensors must be bit-identical to what the stock ``FileSystemReader`` loads, for same-layout checkpoints,
Shard(0) / Shard(1) checkpoints of 2 gloo ranks loaded into full tensors, non-contiguous target views, a mixed plan, a
staging budget smaller than one item and a checkpoint written by ``FileSystemWriterAsync`` on the engine."""
import pytest
import torch
import torch.distributed.checkpoint as dcp
from torch.distributed.checkpoint import DefaultSavePlanner, FileSystemReader

from _mp import run_ranks

pytestmark = pytest.mark.gpu


def _state(device="cuda"):
    g = torch.Generator().manual_seed(3)
    sd = {
        "w": torch.randn(1000, 768, generator=g),
        "b": torch.randn(4099, generator=g).to(torch.bfloat16),
        "ids": torch.randint(0, 1 << 40, (333, 7), generator=g),
        "flags": torch.rand(17, 5, generator=g) > 0.5,
        "c": torch.randn(9, 4, dtype=torch.complex128, generator=g),
        "f8": torch.randn(64, 48, generator=g).to(torch.float8_e4m3fn),
        "step": torch.tensor(7.0),
        "empty": torch.empty(0, 5),
        "t": torch.randn(384, 640, generator=g).t(),  # saved with transposed strides
    }
    return {k: v.to(device) for k, v in sd.items()}


def _targets(like, contiguous=True, device="cuda"):
    out = {}
    for k, v in like.items():
        if contiguous or v.dim() != 2:
            out[k] = torch.zeros(v.shape, dtype=v.dtype, device=device)
        else:
            out[k] = torch.zeros(v.shape[1], v.shape[0], dtype=v.dtype, device=device).t()
    return out


def _stock(path, like):
    out = _targets(like)
    dcp.load(out, storage_reader=FileSystemReader(str(path)))
    return out


def _engine(path, like, contiguous=True):
    from nvidia_resiliency_ext.checkpointing.async_ckpt.cached_metadata_filesystem_reader import CachedMetadataFileSystemReader

    out = _targets(like, contiguous)
    CachedMetadataFileSystemReader.clear_metadata_cache()
    dcp.load(out, storage_reader=CachedMetadataFileSystemReader(str(path), load_on_engine=True))
    torch.cuda.synchronize()
    return out


def _bits(t):
    t = t.detach().contiguous().cpu()
    return bytes(t.reshape(-1).view(torch.uint8).numpy())


def _assert_same(got, ref):
    for k in ref:
        assert got[k].dtype == ref[k].dtype and got[k].shape == ref[k].shape, k
        assert _bits(got[k]) == _bits(ref[k]), k


@pytest.mark.parametrize("contiguous", [True, False])
def test_same_layout_bit_exact(tmp_path, built_library, contiguous):
    from nvidia_resiliency_ext.checkpointing.b200.engine import SnapshotEngine

    sd = _state()
    dcp.save(sd, checkpoint_id=str(tmp_path / "ck"))
    ref = _stock(tmp_path / "ck", sd)
    _assert_same(ref, sd)
    eng = SnapshotEngine.get()
    before = eng.box_batches
    got = _engine(tmp_path / "ck", sd, contiguous)
    assert eng.box_batches > before
    _assert_same(got, ref)


def _shardable(k, v):
    return v.dim() >= 1 and v.numel() and k != "f8"  # gloo's scatter has no float8


def _save_sharded(rank, world, root, placement):
    from torch.distributed.device_mesh import init_device_mesh
    from torch.distributed.tensor import Shard, distribute_tensor

    mesh = init_device_mesh("cpu", (world,))
    sd = {k: distribute_tensor(v.contiguous(), mesh, [Shard(placement if v.dim() > placement else 0)])
          for k, v in _state("cpu").items() if _shardable(k, v)}
    dcp.save(sd, checkpoint_id=root)


@pytest.mark.parametrize("placement", [0, 1])
@pytest.mark.parametrize("contiguous", [True, False])
def test_resharded_two_rank_checkpoint_bit_exact(tmp_path, built_library, placement, contiguous):
    root = str(tmp_path / f"shard{placement}")
    run_ranks(_save_sharded, 2, root, placement)
    full = {k: v.contiguous() for k, v in _state().items() if _shardable(k, v)}
    ref = _stock(root, full)
    _assert_same(ref, full)
    _assert_same(_engine(root, full, contiguous), ref)


def test_mixed_plan(tmp_path, built_library):
    from nvidia_resiliency_ext.checkpointing.async_ckpt.cached_metadata_filesystem_reader import CachedMetadataFileSystemReader

    sd = dict(_state())
    sd["meta"] = {"lr": 0.1, "names": ["a", "b"]}
    dcp.save(sd, checkpoint_id=str(tmp_path / "ck"))
    out = _targets({k: v for k, v in sd.items() if isinstance(v, torch.Tensor)})
    out["meta"] = {"lr": 0.0, "names": []}
    out["ids"] = torch.zeros(sd["ids"].shape, dtype=torch.int64)  # CPU target
    out["w"] = torch.zeros(sd["w"].shape, dtype=torch.float64, device="cuda")  # dtype conversion: stock path
    dcp.load(out, storage_reader=CachedMetadataFileSystemReader(str(tmp_path / "ck"), load_on_engine=True))
    assert out["meta"] == sd["meta"]
    assert torch.equal(out["w"], sd["w"].double()) and torch.equal(out["ids"], sd["ids"].cpu())
    keep = ("b", "flags", "c", "f8", "step", "t")
    _assert_same({k: out[k] for k in keep}, {k: sd[k] for k in keep})


def test_budget_forced_split(tmp_path, built_library, monkeypatch):
    from nvidia_resiliency_ext.checkpointing.b200.engine import SnapshotEngine

    sd = _state()
    dcp.save(sd, checkpoint_id=str(tmp_path / "ck"))
    ref = _stock(tmp_path / "ck", sd)
    monkeypatch.setattr(SnapshotEngine, "DCP_LOAD_STAGING", 256 << 10)  # "w" alone is 3 MB
    got = _engine(tmp_path / "ck", sd, contiguous=False)
    stats = SnapshotEngine.get().last_box_load
    assert stats["batches"] > 10 and stats["peak_staging_bytes"] <= 256 << 10
    _assert_same(got, ref)


def test_checkpoint_written_by_the_async_writer(tmp_path, built_library, dist_1rank):
    from nvidia_resiliency_ext.checkpointing.async_ckpt.core import AsyncCallsQueue, AsyncRequest
    from nvidia_resiliency_ext.checkpointing.async_ckpt.filesystem_async import FileSystemWriterAsync
    from nvidia_resiliency_ext.checkpointing.async_ckpt.state_dict_saver import (
        save_state_dict_async_finalize,
        save_state_dict_async_plan,
    )

    sd = {k: v for k, v in _state().items() if k not in ("t",)}  # the writer snapshots contiguous tensors
    q = AsyncCallsQueue(persistent=False)
    try:
        writer = FileSystemWriterAsync(tmp_path / "ck", thread_count=2)
        ret = save_state_dict_async_plan(sd, writer, None, 0, planner=DefaultSavePlanner())
        save_fn, preload_fn, save_args = writer.get_save_function_and_args()
        q.schedule_async_request(
            AsyncRequest(save_fn, save_args, [lambda ret=ret: save_state_dict_async_finalize(*ret)], preload_fn=preload_fn)
        )
        q.maybe_finalize_async_calls(blocking=True)
    finally:
        q.close()
    ref = _stock(tmp_path / "ck", sd)
    _assert_same(ref, sd)
    _assert_same(_engine(tmp_path / "ck", sd, contiguous=False), ref)
