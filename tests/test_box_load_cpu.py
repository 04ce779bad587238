"""Resharded torch.distributed.checkpoint loads on the engine, without a GPU: the box planner (real library) against the
numpy restatement, the tensor-record parser against torch.load, and ``CachedMetadataFileSystemReader(load_on_engine=True)``
through the fake device layer (which replays the real planner's tiles, tests/_fake_box.py) against the stock ``FileSystemReader``."""
import ctypes as C
import io
import os

import numpy as np
import pytest
import torch
import torch.distributed.checkpoint as dcp

from _box_oracle import _random_boxes, box_copy
from _fake_box import fake_box_device, fake_cuda
from _fake_device import plain
from _mp import run_ranks


# ---------------------------------------------------------------------------------------------------------------------
# planner
# ---------------------------------------------------------------------------------------------------------------------
def _segments(bp):
    """(staging offset, destination address, bytes) of every piece the kernel copies, from the planner's tiles + rows."""
    lib = bp._lib
    out = []
    geo = {}
    for box, row, nrows, off, nby in bp.tiles():
        if box not in geo:
            rb, no, so, dst = C.c_uint64(), C.c_uint32(), C.c_uint64(), C.c_uint64()
            sz, ss, ds = (C.c_uint64 * 8)(), (C.c_int64 * 8)(), (C.c_int64 * 8)()
            assert lib.nvrx_boxplan_box(bp._h, box, C.byref(rb), C.byref(no), sz, ss, ds, C.byref(so), C.byref(dst)) == 0
            k = no.value
            geo[box] = (rb.value, list(sz)[:k], list(ss)[:k], list(ds)[:k], so.value, dst.value)
        rb, sz, ss, ds, so, dst = geo[box]
        for r in range(row, row + nrows):
            s, d, q = so, dst, r
            for k in range(len(sz) - 1, -1, -1):
                q, i = divmod(q, sz[k])
                s += i * ss[k]
                d += i * ds[k]
            lo, n = (off, nby) if nrows == 1 else (0, rb)
            out.append((s + lo, d + lo, n))
    return out


@pytest.mark.parametrize("seed", range(12))
def test_box_planner_matches_box_copy(built_library, seed):
    from nvidia_resiliency_ext.checkpointing.b200.engine import BoxPlan

    rng = np.random.default_rng(seed)
    dst = np.zeros(1 << 20, dtype=np.uint8)
    base = dst.ctypes.data
    boxes, expect, src_bytes, dst_bytes = _random_boxes(rng, int(rng.integers(1, 8)), base)
    assert dst_bytes <= dst.size
    src = rng.integers(0, 256, src_bytes + 1, dtype=np.uint8)
    bp = BoxPlan(boxes, src_bytes, device=0, tile_bytes=4096)
    written = np.zeros(dst.size, dtype=np.int32)
    got = np.zeros_like(dst)
    moved = 0
    for s, d, n in _segments(bp):
        assert 0 <= s and s + n <= src_bytes  # inside staging
        written[d - base : d - base + n] += 1
        got[d - base : d - base + n] = src[s : s + n]
        moved += n
    assert bp.algorithmic_bytes == 2 * moved
    want = np.zeros_like(dst)
    mask = np.zeros(dst.size, dtype=np.int32)
    for elem, sizes, so, sst, do, dstr, _, _ in expect:
        box_copy(src, want, elem, sizes, so, sst, do, dstr)
        ones = np.ones_like(dst)
        probe = np.zeros_like(dst)
        box_copy(ones, probe, elem, sizes, 0, sst, do, dstr)
        mask += probe
        # every source byte the box reads lies inside its extent
    assert np.array_equal(written, mask), "every destination byte exactly once"
    assert np.array_equal(got, want)
    bp.close()


def test_box_planner_long_runs_and_row_groups(built_library):
    from nvidia_resiliency_ext.checkpointing.b200.engine import BoxPlan

    dst = np.zeros(400000, dtype=np.uint8)
    src = np.arange(400000, dtype=np.uint32).astype(np.uint8)
    # a 100000-byte run (split by byte range), 3000-byte rows of a column box, 2-byte rows of a transposed box
    boxes = [
        (1, [100000], 3, [1], dst.ctypes.data + 5, [1]),
        (4, [40, 750], 100003, [1000, 1], dst.ctypes.data + 100100, [800, 1]),
        (2, [30, 20], 300001, [1, 30], dst.ctypes.data + 250001, [20, 1]),
    ]
    bp = BoxPlan(boxes, 400000, device=0, tile_bytes=4096)
    tiles = bp.tiles()
    assert sum(1 for t in tiles if t[0] == 0) == -(-100000 // 4096)  # byte ranges of one row
    assert all(t[2] == 1 for t in tiles if t[0] == 1)  # 3000-byte rows: one per tile
    assert any(t[2] > 1 for t in tiles if t[0] == 2)  # element-wise rows grouped
    want = np.zeros_like(dst)
    for elem, sizes, so, sst, d, dstr in boxes:
        box_copy(src, want, elem, sizes, so, sst, d - dst.ctypes.data, dstr)
    for s, d, n in _segments(bp):
        dst[d - dst.ctypes.data : d - dst.ctypes.data + n] = src[s : s + n]
    assert np.array_equal(dst, want)


def test_box_planner_rejects_malformed_input(built_library):
    from nvidia_resiliency_ext.checkpointing.b200 import _cabi
    from nvidia_resiliency_ext.checkpointing.b200.engine import BoxPlan

    buf = np.zeros(64, dtype=np.uint8)
    p = buf.ctypes.data
    bad = [
        ([(4, [4], 0, [1], p, [1])], 15),  # source byte beyond staging
        ([(4, [1] * 9, 0, [1] * 9, p, [1] * 9)], 64),  # ndim > 8
        ([(3, [4], 0, [1], p, [1])], 64),  # element size
        ([(4, [-1], 0, [1], p, [1])], 64),  # negative size
        ([(4, [2], 0, [-1], p, [1])], 64),  # negative stride
        ([(4, [2], 0, [1], p, [-1])], 64),
    ]
    for boxes, stg in bad:
        with pytest.raises(_cabi.SnapError) as ei:
            BoxPlan(boxes, stg, device=0)
        assert ei.value.status == _cabi.E_INVALID
    ok = BoxPlan([(4, [4], 0, [1], p, [1]), (8, [], 16, [], p + 16, []), (2, [0, 3], 0, [3, 1], 0, [3, 1])], 24, device=0)
    assert ok.algorithmic_bytes == 2 * (16 + 8) and ok.n_tiles == 2


# ---------------------------------------------------------------------------------------------------------------------
# parser
# ---------------------------------------------------------------------------------------------------------------------
_DTYPES = [
    torch.bool, torch.uint8, torch.int8, torch.int16, torch.int32, torch.int64, torch.float16, torch.bfloat16,
    torch.float32, torch.float64, torch.complex64, torch.complex128, torch.float8_e4m3fn, torch.float8_e5m2,
]


@pytest.mark.parametrize("dtype", _DTYPES, ids=str)
def test_tensor_record_parser_agrees_with_torch_load(tmp_path, dtype):
    from nvidia_resiliency_ext.checkpointing.b200.ptzip import read_tensor_record

    g = torch.Generator().manual_seed(1)
    base = (torch.randn(6, 10, generator=g) * 50).to(dtype)
    cases = [base, base[0, 0].clone(), base[:0], base.t(), base[2:5, 1:4].clone(), base.reshape(3, 4, 5).permute(2, 0, 1)]
    path = tmp_path / "chunks.distcp"
    spans = []
    with open(path, "wb") as f:
        for t in cases:
            f.write(b"\0" * 37)
            buf = io.BytesIO()
            torch.save(t, buf)
            spans.append((f.tell(), len(buf.getvalue())))
            f.write(buf.getvalue())
    fd = os.open(path, os.O_RDONLY)
    try:
        for t, (off, length) in zip(cases, spans):
            rec = read_tensor_record(fd, off, length)
            ref = torch.load(io.BytesIO(open(path, "rb").read()[off : off + length]), weights_only=True)
            assert rec.dtype == ref.dtype == dtype
            assert rec.size == tuple(ref.shape) and rec.stride == ref.stride() and rec.storage_offset == ref.storage_offset()
            nbytes = ref.untyped_storage().nbytes()
            assert rec.numel * ref.element_size() == nbytes
            assert os.pread(fd, nbytes, rec.data_off) == bytes(ref.untyped_storage())
        with pytest.raises(ValueError):
            read_tensor_record(fd, 0, spans[0][0] + 10)
    finally:
        os.close(fd)


def test_tensor_record_parser_runs_no_code(tmp_path):
    import pickle

    from nvidia_resiliency_ext.checkpointing.b200.ptzip import read_tensor_record

    class Evil:
        def __reduce__(self):
            return (os.system, ("echo pwned",))

    buf = io.BytesIO()
    torch.save({"x": Evil()}, buf, pickle_module=pickle)
    path = tmp_path / "evil.bin"
    path.write_bytes(buf.getvalue())
    fd = os.open(path, os.O_RDONLY)
    try:
        with pytest.raises(ValueError):
            read_tensor_record(fd, 0, len(buf.getvalue()))
    finally:
        os.close(fd)


# ---------------------------------------------------------------------------------------------------------------------
# reader through the fake device
# ---------------------------------------------------------------------------------------------------------------------
def _state(seed=0):
    g = torch.Generator().manual_seed(seed)
    return {
        "w": torch.randn(64, 96, generator=g),
        "b": torch.randn(96, generator=g).to(torch.bfloat16),
        "ids": torch.randint(0, 1 << 30, (33, 7), generator=g),
        "flags": torch.rand(17, 5, generator=g) > 0.5,
        "c": torch.randn(9, 4, dtype=torch.complex64, generator=g),
        "step": torch.tensor(7.0),
        "empty": torch.empty(0, 5),
        "t": torch.randn(24, 40, generator=g).t(),  # saved with transposed strides
    }


def _stock(path, like):
    out = {k: torch.zeros_like(v) if isinstance(v, torch.Tensor) else v for k, v in like.items()}
    dcp.load(out, storage_reader=dcp.FileSystemReader(str(path)))
    return out


def _engine_load(path, like, *, contiguous=True):
    from nvidia_resiliency_ext.checkpointing.async_ckpt.cached_metadata_filesystem_reader import CachedMetadataFileSystemReader

    out = {}
    for k, v in like.items():
        if not isinstance(v, torch.Tensor):
            out[k] = v
        elif contiguous or v.dim() != 2:
            out[k] = fake_cuda(torch.full_like(v, 3) if v.dtype != torch.bool else torch.zeros_like(v))
        else:
            out[k] = fake_cuda(torch.zeros(v.shape[1], v.shape[0], dtype=v.dtype)).t()  # non-contiguous target view
    CachedMetadataFileSystemReader.clear_metadata_cache()
    dcp.load(out, storage_reader=CachedMetadataFileSystemReader(str(path), load_on_engine=True))
    return out


def _bits_equal(a, b):
    a, b = plain(a).contiguous(), plain(b).contiguous()
    if a.dtype != b.dtype or a.shape != b.shape:
        return False
    return bytes(a.reshape(-1).view(torch.uint8).numpy()) == bytes(b.reshape(-1).view(torch.uint8).numpy())


@pytest.mark.parametrize("contiguous", [True, False])
def test_reader_same_layout_matches_stock(tmp_path, built_library, monkeypatch, contiguous):
    sd = _state()
    dcp.save(sd, checkpoint_id=str(tmp_path / "ck"))
    ref = _stock(tmp_path / "ck", sd)
    with fake_box_device(monkeypatch) as (engine, lib):
        got = _engine_load(tmp_path / "ck", sd, contiguous=contiguous)
        assert "box_scatter" in lib.calls and engine.box_loads == 1
    for k in sd:
        assert _bits_equal(got[k], ref[k]), k


def _save_sharded(rank, world, root, placement):
    from torch.distributed.device_mesh import init_device_mesh
    from torch.distributed.tensor import Shard, distribute_tensor

    mesh = init_device_mesh("cpu", (world,))
    sd = {k: distribute_tensor(v.contiguous(), mesh, [Shard(placement if v.dim() > placement else 0)]) for k, v in _state().items()
          if v.dim() >= 1 and v.numel()}
    dcp.save(sd, checkpoint_id=root)


@pytest.mark.parametrize("placement", [0, 1])
def test_reader_loads_two_rank_shards_into_full_tensors(tmp_path, built_library, monkeypatch, placement):
    root = str(tmp_path / f"shard{placement}")
    run_ranks(_save_sharded, 2, root, placement)
    full = {k: v.contiguous() for k, v in _state().items() if v.dim() >= 1 and v.numel()}
    ref = _stock(root, full)
    for k in full:
        assert _bits_equal(ref[k], full[k]), k
    with fake_box_device(monkeypatch) as (engine, lib):
        got = _engine_load(root, full, contiguous=False)
    for k in full:
        assert _bits_equal(got[k], ref[k]), k


def test_reader_mixed_plan_routes_the_rest_to_the_stock_path(tmp_path, built_library, monkeypatch):
    sd = _state()
    sd["meta"] = {"lr": 0.1, "names": ["a", "b"]}  # BYTE_IO
    dcp.save(sd, checkpoint_id=str(tmp_path / "ck"))
    seen = []
    real = dcp.FileSystemReader.read_data

    def spy(self, plan, planner):
        seen.extend(item.dest_index.fqn for item in plan.items)
        return real(self, plan, planner)

    monkeypatch.setattr(dcp.FileSystemReader, "read_data", spy)
    from nvidia_resiliency_ext.checkpointing.async_ckpt.cached_metadata_filesystem_reader import CachedMetadataFileSystemReader

    with fake_box_device(monkeypatch) as (engine, lib):
        out = {k: fake_cuda(torch.zeros_like(v)) for k, v in sd.items() if isinstance(v, torch.Tensor)}
        out["meta"] = {"lr": 0.0, "names": []}
        out["ids"] = torch.zeros_like(sd["ids"])  # a CPU target
        out["w"] = fake_cuda(torch.zeros(64, 96, dtype=torch.float64))  # dtype differs from the saved one
        dcp.load(out, storage_reader=CachedMetadataFileSystemReader(str(tmp_path / "ck"), load_on_engine=True))
    assert sorted(set(seen)) == ["ids", "meta.lr", "meta.names", "w"] or sorted(set(seen)) == ["ids", "meta", "w"]
    assert out["meta"] == sd["meta"]
    assert torch.equal(plain(out["w"]), sd["w"].double()) and torch.equal(out["ids"], sd["ids"])
    for k in ("b", "flags", "c", "step", "t"):
        assert _bits_equal(out[k], sd[k]), k


def test_reader_budget_smaller_than_one_item_splits(tmp_path, built_library, monkeypatch):
    from nvidia_resiliency_ext.checkpointing.b200.engine import SnapshotEngine

    sd = _state()
    dcp.save(sd, checkpoint_id=str(tmp_path / "ck"))
    ref = _stock(tmp_path / "ck", sd)
    monkeypatch.setattr(SnapshotEngine, "DCP_LOAD_STAGING", 4096)
    with fake_box_device(monkeypatch) as (engine, lib):
        got = _engine_load(tmp_path / "ck", sd, contiguous=False)
        stats = engine.last_box_load
    assert stats["batches"] > 6 and stats["peak_staging_bytes"] <= 4096  # "w" alone is 24 KiB
    for k in sd:
        assert _bits_equal(got[k], ref[k]), k


def test_split_box_pieces_cover_the_box():
    from nvidia_resiliency_ext.checkpointing.b200.engine import box_span, split_box

    sizes, sst, dstr, elem = [5, 7, 9], [70, 1, 7], [63, 9, 1], 4
    seen = set()
    for sz, so, do in split_box(sizes, 3, sst, 0, dstr, elem, 64):
        assert box_span(sz, sst, elem) <= 64
        for i in np.ndindex(*sz):
            s = so + sum(a * b for a, b in zip(i, sst))
            d = do + sum(a * b for a, b in zip(i, dstr))
            assert d not in seen
            seen.add(d)
            assert (s - 3 - sum(a * b for a, b in zip(np.unravel_index(d, (5, 7, 9)), sst))) == 0
    assert len(seen) == 5 * 7 * 9


def test_load_on_engine_without_cuda_raises(tmp_path, built_library):
    from nvidia_resiliency_ext.checkpointing.async_ckpt.cached_metadata_filesystem_reader import CachedMetadataFileSystemReader
    from nvidia_resiliency_ext.checkpointing.b200 import _cabi

    if torch.cuda.is_available():
        pytest.skip("a CUDA device is present")
    with pytest.raises(_cabi.SnapError):
        CachedMetadataFileSystemReader(str(tmp_path), load_on_engine=True)
    CachedMetadataFileSystemReader(str(tmp_path))  # the default stays the stock reader
