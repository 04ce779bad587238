"""GPU tests of verified torch.distributed.checkpoint loads: ``nvrx_crcx_run`` against zlib for extents at every start
residue and many lengths in one launch, ``CachedMetadataFileSystemReader(load_on_engine=True, verify=True)`` bit-equal to
the stock reader (same layout, 2-rank Shard(0) / Shard(1), transposed targets, fp32 -> bf16, a small staging budget, boxes
that do not tile their record, a mixed plan), a flipped byte raising, and the launches the checks add."""
import os
import shutil
import warnings
import zlib

import numpy as np
import pytest
import torch
import torch.distributed.checkpoint as dcp
from torch.distributed.checkpoint import FileSystemReader
from torch.distributed.checkpoint.api import CheckpointException

from _mp import run_ranks

pytestmark = pytest.mark.gpu

LENGTHS = [0, 1, 15, 16, 17, 511, 512, 513, 65535, 65536, 65537, 3 * 65536 + 519, (16 << 20) + 5]
SENTINEL = 0x5A5A5A5A


def _run_extents(buf_dev, offsets, nbytes):
    from nvidia_resiliency_ext.checkpointing.b200.engine import CrcxPlan

    plan = CrcxPlan(offsets, nbytes, torch.cuda.current_device())
    host = torch.full((len(offsets) + 8,), SENTINEL, dtype=torch.int32).pin_memory()
    plan.run(buf_dev.data_ptr(), host.data_ptr(), torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    vals = [v & 0xFFFFFFFF for v in host.tolist()]
    launches = plan.launches
    plan.close()
    return vals[: len(offsets)], vals[len(offsets):], launches


def test_crcx_matches_zlib_at_every_residue(built_library):
    rng = np.random.default_rng(0)
    offsets, nbytes, cur = [], [], 0
    for length in LENGTHS:
        for res in range(16):
            cur = -(-cur // 16) * 16 + res + int(rng.integers(0, 3)) * 16
            offsets.append(cur)
            nbytes.append(length)
            cur += length
    data = rng.integers(0, 256, cur + 64, dtype=np.uint8)
    data[1000:5000] = 0xFF
    dev = torch.from_numpy(data).cuda()
    got, past, launches = _run_extents(dev, offsets, nbytes)
    want = [zlib.crc32(data[o:o + n].tobytes()) for o, n in zip(offsets, nbytes)]
    bad = [(o % 16, n) for o, n, g, w in zip(offsets, nbytes, got, want) if g != w]
    assert not bad, bad[:10]
    assert past == [SENTINEL] * 8 and launches == 2


def test_crcx_back_to_back_and_overlapping_extents(built_library):
    rng = np.random.default_rng(1)
    data = rng.integers(0, 256, 3 << 20, dtype=np.uint8)
    dev = torch.from_numpy(data).cuda()
    cuts = np.sort(rng.choice(np.arange(1, len(data)), 200, replace=False))
    edges = [0, *cuts.tolist(), len(data)]
    offsets = edges[:-1] + [3, 0, 100_003]
    nbytes = [b - a for a, b in zip(edges, edges[1:])] + [2_000_000, len(data), 7]
    got, past, _ = _run_extents(dev, offsets, nbytes)
    assert got == [zlib.crc32(data[o:o + n].tobytes()) for o, n in zip(offsets, nbytes)]
    assert past == [SENTINEL] * 8
    # only sub-row extents: one launch
    got, _, launches = _run_extents(dev, [5, 40, 999], [300, 0, 511])
    assert launches == 1 and got == [zlib.crc32(data[o:o + n].tobytes()) for o, n in zip([5, 40, 999], [300, 0, 511])]


# ---------------------------------------------------------------------------------------------------------------------
# the reader
# ---------------------------------------------------------------------------------------------------------------------
def _state(device="cuda"):
    g = torch.Generator().manual_seed(3)
    sd = {
        "w": torch.randn(1000, 768, generator=g),
        "b": torch.randn(4099, generator=g).to(torch.bfloat16),
        "ids": torch.randint(0, 1 << 40, (333, 7), generator=g),
        "flags": torch.rand(17, 5, generator=g) > 0.5,
        "step": torch.tensor(7.0),
        "empty": torch.empty(0, 5),
        "t": torch.randn(384, 640, generator=g).t(),  # saved with transposed strides
    }
    return {k: v.to(device) for k, v in sd.items()}


N_RECORDS = 6


def _targets(like, contiguous=True, dtype=None):
    out = {}
    for k, v in like.items():
        dt = dtype if (dtype is not None and v.dtype == torch.float32) else v.dtype
        if contiguous or v.dim() != 2:
            out[k] = torch.zeros(v.shape, dtype=dt, device="cuda")
        else:
            out[k] = torch.zeros(v.shape[1], v.shape[0], dtype=dt, device="cuda").t()
    return out


def _stock(path, like, dtype=None):
    out = _targets(like, dtype=dtype)
    dcp.load(out, storage_reader=FileSystemReader(str(path)))
    return out


def _verified(path, like, contiguous=True, dtype=None):
    from nvidia_resiliency_ext.checkpointing.async_ckpt.cached_metadata_filesystem_reader import CachedMetadataFileSystemReader
    from nvidia_resiliency_ext.checkpointing.b200.engine import SnapshotEngine

    out = _targets(like, contiguous, dtype)
    CachedMetadataFileSystemReader.clear_metadata_cache()
    reader = CachedMetadataFileSystemReader(str(path), load_on_engine=True, verify=True)
    with warnings.catch_warnings(record=True) as seen:
        warnings.simplefilter("always")
        dcp.load(out, storage_reader=reader)
    assert not [w for w in seen if "checksum" in str(w.message)]
    torch.cuda.synchronize()
    return out, dict(SnapshotEngine.get().last_box_load), reader


def _bits(t):
    t = t.detach().contiguous().cpu()
    return bytes(t.reshape(-1).view(torch.uint8).numpy())


def _assert_same(got, ref):
    for k in ref:
        assert got[k].dtype == ref[k].dtype and got[k].shape == ref[k].shape, k
        assert _bits(got[k]) == _bits(ref[k]), k


@pytest.mark.parametrize("contiguous", [True, False])
def test_verified_same_layout_bit_exact(tmp_path, built_library, contiguous):
    sd = _state()
    dcp.save(sd, checkpoint_id=str(tmp_path / "ck"))
    ref = _stock(tmp_path / "ck", sd)
    got, stats, reader = _verified(tmp_path / "ck", sd, contiguous)
    _assert_same(got, ref)
    assert stats["verified_records"] == N_RECORDS and stats["verify_extra_bytes"] == 0 and stats["unverified_records"] == 0
    assert reader.last_verify == {"gpu_records": N_RECORDS, "host_records": 0, "unverified": 0}


def _save_sharded(rank, world, root, placement):
    from torch.distributed.device_mesh import init_device_mesh
    from torch.distributed.tensor import Shard, distribute_tensor

    mesh = init_device_mesh("cpu", (world,))
    sd = {k: distribute_tensor(v.contiguous(), mesh, [Shard(placement if v.dim() > placement else 0)])
          for k, v in _state("cpu").items() if v.dim() >= 1 and v.numel()}
    dcp.save(sd, checkpoint_id=root)


@pytest.mark.parametrize("placement", [0, 1])
def test_verified_two_rank_shards_bit_exact(tmp_path, built_library, placement):
    root = str(tmp_path / f"shard{placement}")
    run_ranks(_save_sharded, 2, root, placement)
    full = {k: v.contiguous() for k, v in _state().items() if v.dim() >= 1 and v.numel()}
    ref = _stock(root, full)
    got, stats, _ = _verified(root, full, contiguous=False)
    _assert_same(got, ref)
    assert stats["verified_records"] == 2 * len(full) and stats["verify_extra_bytes"] == 0


def test_verified_fp32_to_bf16_small_budget(tmp_path, built_library, monkeypatch):
    from nvidia_resiliency_ext.checkpointing.b200.engine import SnapshotEngine

    sd = _state()
    dcp.save(sd, checkpoint_id=str(tmp_path / "ck"))
    ref = _stock(tmp_path / "ck", sd, dtype=torch.bfloat16)
    for budget in (SnapshotEngine.DCP_LOAD_STAGING, 1 << 20, 64 << 10):
        monkeypatch.setattr(SnapshotEngine, "DCP_LOAD_STAGING", budget)
        got, stats, _ = _verified(tmp_path / "ck", sd, contiguous=False, dtype=torch.bfloat16)
        _assert_same(got, ref)
        # below its 960 KiB, the transposed "t" is cut along its stride-1 dim: the pieces' spans interleave, so its record
        # is read once more, whole, for the check; every other record is tiled by its pieces
        extra = 384 * 640 * 4 if budget < 384 * 640 * 4 + 16 else 0
        assert stats["verified_records"] == N_RECORDS and stats["verify_extra_bytes"] == extra, budget
        if budget == 64 << 10:
            assert stats["batches"] > 40  # "w" alone is 3 MB: records are chained over batches


def test_verified_boxes_that_do_not_tile_their_record(tmp_path, built_library):
    from nvidia_resiliency_ext.checkpointing.b200._cabi import SnapError
    from nvidia_resiliency_ext.checkpointing.b200.engine import BoxLoad, SnapshotEngine
    from nvidia_resiliency_ext.checkpointing.b200.ptzip import read_tensor_record

    w = torch.randn(1000, 768)
    dcp.save({"w": w}, checkpoint_id=str(tmp_path / "ck"))
    md = FileSystemReader(str(tmp_path / "ck")).read_metadata()
    (idx, item), = md.storage_data.items()
    path = os.path.join(str(tmp_path / "ck"), item.relative_path)
    fd = os.open(path, os.O_RDONLY)
    rec = read_tensor_record(fd, item.offset, item.length)
    os.close(fd)
    engine = SnapshotEngine.get()
    L = rec.record_len
    for boxes, shapes, extra in (
        ([(0, 0)], [(1000, 384)], 384 * 4),                            # columns 0-383 of every row: the tail is added
        ([(0, 0), (0, 384)], [(1000, 384), (1000, 384)], L),          # interleaved spans: the record once more
        ([(0, 0), (999, 0)], [(1, 768), (1, 768)], 998 * 768 * 4),     # first and last rows: the gap is read for the check
    ):
        targets = [torch.zeros(s, device="cuda") for s in shapes]
        assert tuple(rec.stride) == (768, 1)
        entries = [BoxLoad(path, rec.data_off, rec.numel * 4, rec.storage_offset + r0 * 768 + c0, rec.stride, t, record_crc=rec.crc32,
                           record_len=L, name="w") for (r0, c0), t in zip(boxes, targets)]
        engine.load_boxes(entries, verify=True)
        stats = engine.last_box_load
        assert stats["verified_records"] == 1 and stats["verify_extra_bytes"] == extra and stats["crc_bytes"] == L
        for (r0, c0), s, t in zip(boxes, shapes, targets):
            assert torch.equal(t.cpu(), w[r0:r0 + s[0], c0:c0 + s[1]])
        with pytest.raises(SnapError, match="crc32 mismatch"):
            engine.load_boxes([e._replace(record_crc=rec.crc32 ^ 0x80) for e in entries], verify=True)


def test_verified_mixed_plan(tmp_path, built_library):
    from nvidia_resiliency_ext.checkpointing.async_ckpt.cached_metadata_filesystem_reader import CachedMetadataFileSystemReader

    sd = _state()
    sd["meta"] = {"lr": 0.1, "names": ["a", "b"]}
    dcp.save(sd, checkpoint_id=str(tmp_path / "ck"))
    out = _targets({k: v for k, v in sd.items() if isinstance(v, torch.Tensor)})
    out["meta"] = {"lr": 0.0, "names": []}
    out["ids"] = torch.zeros(sd["ids"].shape, dtype=sd["ids"].dtype)  # CPU target: checked on the host
    CachedMetadataFileSystemReader.clear_metadata_cache()
    reader = CachedMetadataFileSystemReader(str(tmp_path / "ck"), load_on_engine=True, verify=True)
    with pytest.warns(UserWarning, match="without a checksum check"):
        dcp.load(out, storage_reader=reader)
    assert reader.last_verify["host_records"] == 1 and reader.last_verify["gpu_records"] == N_RECORDS - 1
    assert out["meta"] == sd["meta"] and torch.equal(out["ids"], sd["ids"].cpu())
    for k in ("w", "b", "flags", "step", "t"):
        assert _bits(out[k]) == _bits(sd[k]), k


@pytest.mark.parametrize("fqn", ["w", "t"])
def test_flipped_byte_raises(tmp_path, built_library, fqn):
    from nvidia_resiliency_ext.checkpointing.async_ckpt.cached_metadata_filesystem_reader import CachedMetadataFileSystemReader
    from nvidia_resiliency_ext.checkpointing.b200.ptzip import read_tensor_record

    sd = _state()
    dcp.save(sd, checkpoint_id=str(tmp_path / "ck"))
    shutil.copytree(tmp_path / "ck", tmp_path / "bad")
    md = FileSystemReader(str(tmp_path / "bad")).read_metadata()
    item = next(v for k, v in md.storage_data.items() if k.fqn == fqn)
    path = os.path.join(str(tmp_path / "bad"), item.relative_path)
    fd = os.open(path, os.O_RDWR)
    try:
        rec = read_tensor_record(fd, item.offset, item.length)
        at = rec.data_off + rec.record_len - 3  # in the tail of the record
        os.pwrite(fd, bytes([os.pread(fd, 1, at)[0] ^ 0x01]), at)
    finally:
        os.close(fd)
    CachedMetadataFileSystemReader.clear_metadata_cache()
    with pytest.raises(CheckpointException, match=rf"(?s)crc32 mismatch on 1 of {N_RECORDS} records \({fqn} in "):
        dcp.load(_targets(sd), storage_reader=CachedMetadataFileSystemReader(str(tmp_path / "bad"), load_on_engine=True, verify=True))


def test_verify_adds_exactly_the_crc_launches(tmp_path, built_library, monkeypatch):
    from nvidia_resiliency_ext.checkpointing.async_ckpt.cached_metadata_filesystem_reader import CachedMetadataFileSystemReader
    from nvidia_resiliency_ext.checkpointing.b200.engine import CrcxPlan, SnapshotEngine

    sd = _state()
    dcp.save(sd, checkpoint_id=str(tmp_path / "ck"))
    engine = SnapshotEngine.get()
    crc_launches = []
    real_run = CrcxPlan.run
    monkeypatch.setattr(CrcxPlan, "run", lambda self, *a: (crc_launches.append(self.launches), real_run(self, *a))[1])
    default = SnapshotEngine.DCP_LOAD_STAGING
    for budget in (default, 256 << 10):
        monkeypatch.setattr(SnapshotEngine, "DCP_LOAD_STAGING", budget)
        counts = {}
        for verify in (False, True):
            crc_launches.clear()
            CachedMetadataFileSystemReader.clear_metadata_cache()
            before = engine.launches
            dcp.load(_targets(sd), storage_reader=CachedMetadataFileSystemReader(str(tmp_path / "ck"), load_on_engine=True, verify=verify))
            counts[verify] = (engine.launches - before, engine.last_box_load["batches"], list(crc_launches))
        (plain, batches, none), (checked, vbatches, runs) = counts[False], counts[True]
        # one checksum run per batch that holds checked bytes.  At the small budget the transposed "t" is cut into pieces
        # whose spans interleave: they stay unchecked and its record is read once more, whole, in extra batches
        assert none == [] and 0 < len(runs) <= vbatches
        if budget == default:
            assert batches == vbatches == len(runs)
        assert checked - plain == sum(runs) and all(r in (1, 2) for r in runs)
