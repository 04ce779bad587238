"""Verified torch.distributed.checkpoint loads, everything that can be checked without a GPU: the CRC arithmetic of
``nvrx_crcx_run`` driven on the host (tests/crcx_lanes.cpp) and ``nvrx_crc32_combine`` against zlib, the read-range planning
of ``load_boxes(verify=True)``, and ``CachedMetadataFileSystemReader(verify=True)`` through the fake device layer, whose
stand-in for ``nvrx_crcx_run`` sums the fake staging as the gap-poisoning fill left it (a misplaced range fails)."""
import contextlib
import ctypes as C
import ctypes.util
import os
import shutil
import subprocess
import types
import warnings
import zlib

import numpy as np
import pytest
import torch
import torch.distributed.checkpoint as dcp

from _box_oracle import _random_boxes
from _fake_box import fake_box_device, fake_cuda
from _fake_device import _val, plain
from _mp import run_ranks
from conftest import ROOT


# ---------------------------------------------------------------------------------------------------------------------
# arithmetic
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def lanes(tmp_path_factory):
    out = tmp_path_factory.mktemp("crcx") / "libcrcx_lanes.so"
    res = subprocess.run(
        ["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-x", "c++", f"-I{ROOT / 'nvidia-resiliency-ext_b200' / 'csrc'}",
         "-o", str(out), str(ROOT / "tests" / "crcx_lanes.cpp")],
        capture_output=True, text=True,
    )
    assert res.returncode == 0, res.stdout + res.stderr
    lib = C.CDLL(str(out))
    lib.crcx_lanes_extent.restype = C.c_uint32
    lib.crcx_lanes_extent.argtypes = [C.c_void_p, C.c_uint64, C.c_uint64]
    lib.crcx_lanes_pow2.restype = None
    lib.crcx_lanes_pow2.argtypes = [C.c_void_p]
    return lib


def _operator(which):
    from nvidia_resiliency_ext.checkpointing.b200 import _cabi

    out = (C.c_uint32 * 1024)()
    _cabi.check(_cabi.lib().nvrx_crc_operator(which, out), "nvrx_crc_operator")
    return np.frombuffer(out, dtype=np.uint32).copy()


def test_pow2_tables_are_the_library_operators(built_library, lanes):
    pow2 = np.zeros(64 * 1024, dtype=np.uint32)
    lanes.crcx_lanes_pow2(pow2.ctypes.data)
    for k, which in ((2, 4), (4, 16), (9, 512), (16, 0)):
        assert np.array_equal(pow2[k * 1024:(k + 1) * 1024], _operator(which)), which


LENGTHS = [0, 1, 2, 15, 16, 17, 31, 32, 33, 496, 511, 512, 513, 527, 528, 1023, 1024 + 7, 65535, 65536, 65537,
           65536 + 512 + 3, 3 * 65536 + 519, 33 * 65536 + 100]


def test_head_body_tail_arithmetic_matches_zlib(lanes):
    rng = np.random.default_rng(11)
    buf = rng.integers(0, 256, 33 * 65536 + 200, dtype=np.uint8)
    buf[100:700] = 0xFF  # runs of equal bytes, too
    for length in LENGTHS:
        for res in range(16):
            off = 16 * 3 + res
            got = lanes.crcx_lanes_extent(buf.ctypes.data, off, length)
            assert got == zlib.crc32(buf[off:off + length].tobytes()), (res, length)


def test_combine_matches_zlib(built_library):
    from nvidia_resiliency_ext.checkpointing.b200.engine import crc32_combine

    rng = np.random.default_rng(2)
    data = rng.integers(0, 256, 200_000, dtype=np.uint8).tobytes()
    for cut in [0, 1, 2, 15, 16, 511, 512, 65536, len(data) - 1, len(data)] + [int(x) for x in rng.integers(0, len(data), 20)]:
        a, b = data[:cut], data[cut:]
        assert crc32_combine(zlib.crc32(a), zlib.crc32(b), len(b)) == zlib.crc32(data), cut
    assert crc32_combine(0x12345678, 0, 0) == 0x12345678
    assert crc32_combine(zlib.crc32(b"abc"), zlib.crc32(b"d"), 1) == zlib.crc32(b"abcd")


def test_combine_of_long_lengths_matches_system_zlib(built_library):
    from nvidia_resiliency_ext.checkpointing.b200.engine import crc32_combine

    name = ctypes.util.find_library("z")
    if name is None:
        pytest.skip("no system libz")
    libz = C.CDLL(name)
    libz.crc32_combine64.restype = C.c_ulong
    libz.crc32_combine64.argtypes = [C.c_ulong, C.c_ulong, C.c_int64]
    rng = np.random.default_rng(4)
    lens = [2, 3, (1 << 32) - 1, 1 << 32, (1 << 32) + 17, 1 << 40, (1 << 40) - 5] + [int(x) for x in rng.integers(1, 1 << 40, 20)]
    for n in lens:
        a, b = int(rng.integers(0, 1 << 32)), int(rng.integers(0, 1 << 32))
        assert crc32_combine(a, b, n) == libz.crc32_combine64(a, b, n), n


def test_crcx_create_rejects_bad_input_and_counts_work(built_library):
    from nvidia_resiliency_ext.checkpointing.b200 import _cabi
    from nvidia_resiliency_ext.checkpointing.b200.engine import CrcxPlan

    lib = _cabi.lib()
    h = C.c_void_p()
    assert lib.nvrx_crcx_create(2, None, None, 0, C.byref(h)) == _cabi.E_INVALID
    u64 = lambda *v: (C.c_uint64 * len(v))(*v)  # noqa: E731
    assert lib.nvrx_crcx_create(1, u64((1 << 64) - 8), u64(9), 0, C.byref(h)) == _cabi.E_INVALID
    assert lib.nvrx_crcx_create(-1, u64(0), u64(0), 0, C.byref(h)) == _cabi.E_INVALID
    plan = CrcxPlan([3, 0, 100], [5, 0, 64 + 3 * 65536 + 512 * 5 + 7], 0)  # sub-row, empty, head + 3 chunks + 1 + tail
    assert (plan.n_chunks, plan.launches) == (4, 2)
    plan.close()
    plan = CrcxPlan([1], [600], 0)  # head 15 + one row + tail
    assert (plan.n_chunks, plan.launches) == (1, 2)
    plan.close()
    plan = CrcxPlan([7], [300], 0)
    assert (plan.n_chunks, plan.launches) == (0, 1)
    plan.close()
    plan = CrcxPlan([], [], 0)
    assert (plan.n_chunks, plan.launches) == (0, 0)
    assert lib.nvrx_crcx_run(plan._h, None, None, None) == 0  # nothing to do
    plan.close()


# ---------------------------------------------------------------------------------------------------------------------
# read-range planning
# ---------------------------------------------------------------------------------------------------------------------
def _check_ranges(spans, length, limit):
    from nvidia_resiliency_ext.checkpointing.b200.engine import record_verify_ranges

    ranges, whole = record_verify_ranges(spans, length, limit)
    assert all(0 < e - r <= limit for r, e in whole)
    srt = sorted(spans)
    overlap = any(b[0] < a[1] for a, b in zip(srt, srt[1:]))
    if ranges is None:
        assert overlap
        cover = sorted(whole)
    else:
        assert not overlap and len(ranges) == len(spans)
        for (a, b), (r, e) in zip(spans, ranges):
            assert r <= a and b <= e and e - r <= max(limit, b - a)
        cover = sorted(list(ranges) + list(whole))
    pos = 0
    for r, e in cover:  # tiles [0, length) exactly once
        assert r == pos and e >= r
        pos = e
    assert pos == length
    return ranges, whole


def test_verify_ranges_tile_the_record_on_random_boxes():
    from nvidia_resiliency_ext.checkpointing.b200.engine import box_span, split_box

    rng = np.random.default_rng(7)
    tiled = 0
    for seed in range(40):
        _, expect, src_bytes, _ = _random_boxes(rng, int(rng.integers(1, 6)), 0)
        length = src_bytes + int(rng.integers(0, 50))
        for budget in (1 << 20, 4096, 512, 96):
            spans = []
            for elem, sizes, src_off, sst, _, _, _, _ in expect:
                if box_span(sizes, sst, elem) == 0:
                    continue
                for sz, so, _ in split_box(sizes, 0, sst, 0, sst, elem, budget - 16):
                    a = src_off + so * elem
                    spans.append((a, a + box_span(sz, sst, elem)))
            if spans:
                _check_ranges(spans, length, budget - 16)
        # pieces that already tile a record: no extra byte, whatever the budget
        cuts = sorted(set(int(x) for x in rng.integers(1, length, int(rng.integers(0, 6))))) if length > 1 else []
        edges = [0] + cuts + [length]
        spans = [(a, b) for a, b in zip(edges, edges[1:])]
        perm = [spans[i] for i in rng.permutation(len(spans))]
        ranges, whole = _check_ranges(perm, length, max(b - a for a, b in spans))
        assert whole == [] and list(ranges) == perm
        tiled += 1
    assert tiled == 40


def test_verify_ranges_examples():
    # a column box of a 4 x 8 record of 4-byte elements: columns 0-3 read [0, 112); the tail [112, 128) is added
    ranges, whole = _check_ranges([(0, 112)], 128, 1 << 20)
    assert ranges == [(0, 128)] and whole == []
    # a record read by two entries with a gap: the first range reaches the second span
    ranges, whole = _check_ranges([(64, 100), (10, 20)], 128, 1 << 20)
    assert ranges == [(64, 128), (0, 64)] and whole == []
    # overlapping spans: the record is read once more, whole, in parts that fit the limit
    ranges, whole = _check_ranges([(0, 64), (32, 100)], 128, 50)
    assert ranges is None and whole == [(0, 50), (50, 100), (100, 128)]
    # a gap too long for one batch travels on its own
    ranges, whole = _check_ranges([(0, 10), (200, 210)], 300, 64)
    assert ranges == [(0, 10), (200, 210)]


# ---------------------------------------------------------------------------------------------------------------------
# reader through the fake device
# ---------------------------------------------------------------------------------------------------------------------
def _crcx_create(self, n, offsets, nbytes, device, out):
    rc = self._real.nvrx_crcx_create(n, offsets, nbytes, device, out)
    if rc == 0:
        self._crcx[out._obj.value] = ([offsets[i] for i in range(n)], [nbytes[i] for i in range(n)])
    return rc


def _crcx_run(self, h, base, host, stream):
    offs, nbs = self._crcx[_val(h)]
    vals = [zlib.crc32(C.string_at(_val(base) + o, n)) for o, n in zip(offs, nbs)]
    if vals:
        C.memmove(_val(host), (C.c_uint32 * len(vals))(*vals), 4 * len(vals))
    self.calls.append("crcx")
    return 0


@contextlib.contextmanager
def fake_crc_device(monkeypatch, base=fake_box_device):
    """``fake_box_device`` (or the converting one) plus a stand-in for ``nvrx_crcx_run``: zlib over the fake staging at the
    planned extents."""
    with base(monkeypatch) as (engine, lib):
        lib._crcx = {}
        lib.nvrx_crcx_create = types.MethodType(_crcx_create, lib)
        lib.nvrx_crcx_run = types.MethodType(_crcx_run, lib)
        lib.nvrx_crcx_commit = lambda h, stream: 0
        yield engine, lib


def _state(seed=0):
    g = torch.Generator().manual_seed(seed)
    return {
        "w": torch.randn(64, 96, generator=g),
        "b": torch.randn(96, generator=g).to(torch.bfloat16),
        "ids": torch.randint(0, 1 << 30, (33, 7), generator=g),
        "flags": torch.rand(17, 5, generator=g) > 0.5,
        "step": torch.tensor(7.0),
        "empty": torch.empty(0, 5),
        "t": torch.randn(24, 40, generator=g).t(),  # saved with transposed strides
    }


N_RECORDS = 6  # non-empty tensors of _state()


def _stock(path, like):
    out = {k: torch.zeros_like(v) if isinstance(v, torch.Tensor) else v for k, v in like.items()}
    dcp.load(out, storage_reader=dcp.FileSystemReader(str(path)))
    return out


def _reader(path, **kw):
    from nvidia_resiliency_ext.checkpointing.async_ckpt.cached_metadata_filesystem_reader import CachedMetadataFileSystemReader

    CachedMetadataFileSystemReader.clear_metadata_cache()
    return CachedMetadataFileSystemReader(str(path), **kw)


def _targets(like, *, contiguous=True, dtype=None):
    out = {}
    for k, v in like.items():
        if not isinstance(v, torch.Tensor):
            out[k] = v
            continue
        dt = dtype if (dtype is not None and v.dtype == torch.float32) else v.dtype
        if contiguous or v.dim() != 2:
            out[k] = fake_cuda(torch.full(v.shape, 3, dtype=dt) if dt != torch.bool else torch.zeros(v.shape, dtype=dt))
        else:
            out[k] = fake_cuda(torch.zeros(v.shape[1], v.shape[0], dtype=dt)).t()
    return out


def _bits_equal(a, b):
    a, b = plain(a).contiguous(), plain(b).contiguous()
    if a.dtype != b.dtype or a.shape != b.shape:
        return False
    return bytes(a.reshape(-1).view(torch.uint8).numpy()) == bytes(b.reshape(-1).view(torch.uint8).numpy())


def _verified_load(path, like, monkeypatch, base=fake_box_device, **kw):
    with fake_crc_device(monkeypatch, base) as (engine, lib):
        reader = _reader(path, load_on_engine=True, verify=True)
        out = _targets(like, **kw)
        with warnings.catch_warnings(record=True) as seen:
            warnings.simplefilter("always")
            dcp.load(out, storage_reader=reader)
        assert not [w for w in seen if "checksum" in str(w.message)]  # every record here carries one
        stats, calls = dict(engine.last_box_load), list(lib.calls)
    return out, stats, calls, reader


@pytest.mark.parametrize("contiguous", [True, False])
def test_verified_same_layout_matches_stock(tmp_path, built_library, monkeypatch, contiguous):
    sd = _state()
    dcp.save(sd, checkpoint_id=str(tmp_path / "ck"))
    ref = _stock(tmp_path / "ck", sd)
    got, stats, calls, reader = _verified_load(tmp_path / "ck", sd, monkeypatch, contiguous=contiguous)
    assert stats["verified_records"] == N_RECORDS and stats["unverified_records"] == 0 and stats["verify_extra_bytes"] == 0
    assert calls.count("crcx") == stats["batches"] == 1
    assert reader.last_verify == {"gpu_records": N_RECORDS, "host_records": 0, "unverified": 0}
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
def test_verified_two_rank_shards_into_full_tensors(tmp_path, built_library, monkeypatch, placement):
    root = str(tmp_path / f"shard{placement}")
    run_ranks(_save_sharded, 2, root, placement)
    full = {k: v.contiguous() for k, v in _state().items() if v.dim() >= 1 and v.numel()}
    ref = _stock(root, full)
    got, stats, _, _ = _verified_load(root, full, monkeypatch, contiguous=False)
    assert stats["verified_records"] == 2 * len(full) and stats["verify_extra_bytes"] == 0
    for k in full:
        assert _bits_equal(got[k], ref[k]), k


def test_verified_converting_items_are_checked_as_stored(tmp_path, built_library, monkeypatch):
    sd = {k: v for k, v in _state().items() if v.dtype == torch.float32}
    dcp.save(sd, checkpoint_id=str(tmp_path / "ck"))
    ref = {k: v.to(torch.bfloat16) for k, v in sd.items()}
    from test_box_cast_cpu import fake_cast_box_device

    got, stats, _, _ = _verified_load(tmp_path / "ck", sd, monkeypatch, fake_cast_box_device, contiguous=False, dtype=torch.bfloat16)
    assert stats["verified_records"] == sum(1 for v in sd.values() if v.numel()) and stats["verify_extra_bytes"] == 0
    for k in sd:
        assert _bits_equal(got[k], ref[k]), k


def test_verified_tiny_budget_chains_records_over_batches(tmp_path, built_library, monkeypatch):
    from nvidia_resiliency_ext.checkpointing.b200.engine import SnapshotEngine

    sd = _state()
    dcp.save(sd, checkpoint_id=str(tmp_path / "ck"))
    ref = _stock(tmp_path / "ck", sd)
    monkeypatch.setattr(SnapshotEngine, "DCP_LOAD_STAGING", 4096)
    got, stats, calls, _ = _verified_load(tmp_path / "ck", sd, monkeypatch, contiguous=False)
    assert stats["batches"] > 6 and stats["peak_staging_bytes"] <= 4096  # "w" alone is 24 KiB
    assert stats["verified_records"] == N_RECORDS and stats["verify_extra_bytes"] == 0
    assert calls.count("crcx") == stats["batches"]
    for k in sd:
        assert _bits_equal(got[k], ref[k]), k


def _record(path):
    """(file, record offset, record length, crc) of the single tensor item ``w`` of a one-rank checkpoint."""
    from nvidia_resiliency_ext.checkpointing.b200.ptzip import read_tensor_record

    reader = dcp.FileSystemReader(str(path))
    md = reader.read_metadata()
    info = md.storage_data
    out = {}
    for idx, item in info.items():
        f = os.path.join(str(path), item.relative_path)
        fd = os.open(f, os.O_RDONLY)
        try:
            out[idx.fqn] = (f, read_tensor_record(fd, item.offset, item.length))
        finally:
            os.close(fd)
    return out


def _entries_for(path, fqn, boxes, targets):
    """BoxLoads of sub-boxes (start row, start col) of the saved 2-d item ``fqn`` into ``targets``."""
    from nvidia_resiliency_ext.checkpointing.b200.engine import BoxLoad

    f, rec = _record(path)[fqn]
    out = []
    for (r0, c0), t in zip(boxes, targets):
        src_off = rec.storage_offset + r0 * rec.stride[0] + c0 * rec.stride[1]
        out.append(BoxLoad(f, rec.data_off, rec.numel * rec.dtype.itemsize, src_off, rec.stride, t,
                           record_crc=rec.crc32, record_len=rec.record_len, name=fqn))
    return out, rec


@pytest.mark.parametrize("case", ["columns", "row_halves", "column_halves", "far_rows"])
def test_verified_boxes_that_do_not_tile_their_record(tmp_path, built_library, monkeypatch, case):
    from nvidia_resiliency_ext.checkpointing.b200._cabi import SnapError
    from nvidia_resiliency_ext.checkpointing.b200.engine import SnapshotEngine

    w = torch.randn(64, 96, generator=torch.Generator().manual_seed(5))
    dcp.save({"w": w}, checkpoint_id=str(tmp_path / "ck"))
    if case == "columns":  # a Shard(1)-like target: columns 0..47 of every row -> the record's tail is added
        boxes, shapes, expect_extra = [(0, 0)], [(64, 48)], 4 * 48
    elif case == "row_halves":  # two entries, rows 0-31 and 32-63: together they tile the record
        boxes, shapes, expect_extra = [(0, 0), (32, 0)], [(32, 96), (32, 96)], 0
    elif case == "column_halves":  # two entries whose spans interleave: the record is read once more, whole
        boxes, shapes, expect_extra = [(0, 0), (0, 48)], [(64, 48), (64, 48)], 64 * 96 * 4
    else:  # first and last rows with a 4 KiB budget: the gap travels in checksum-only reads
        boxes, shapes, expect_extra = [(0, 0), (63, 0)], [(1, 96), (1, 96)], 62 * 96 * 4
        monkeypatch.setattr(SnapshotEngine, "DCP_LOAD_STAGING", 4096)
    with fake_crc_device(monkeypatch) as (engine, lib):
        targets = [fake_cuda(torch.zeros(s)) for s in shapes]
        entries, rec = _entries_for(tmp_path / "ck", "w", boxes, targets)
        engine.load_boxes(entries, verify=True)
        stats = engine.last_box_load
        assert stats["verified_records"] == 1 and stats["verify_extra_bytes"] == expect_extra
        assert stats["crc_bytes"] == rec.record_len == 64 * 96 * 4  # every byte of the record summed once
        for (r0, c0), s, t in zip(boxes, shapes, targets):
            assert torch.equal(plain(t), w[r0:r0 + s[0], c0:c0 + s[1]]), case
        # the same load against a wrong checksum fails, naming the item
        bad = [e._replace(record_crc=rec.crc32 ^ 1) for e in entries]
        with pytest.raises(SnapError, match=r"crc32 mismatch on 1 of 1 records \(w in .* at record offset"):
            engine.load_boxes(bad, verify=True)


def test_verified_mixed_plan_checks_stock_items_on_the_host(tmp_path, built_library, monkeypatch):
    sd = _state()
    sd["meta"] = {"lr": 0.1, "names": ["a", "b"]}  # BYTE_IO
    dcp.save(sd, checkpoint_id=str(tmp_path / "ck"))
    with fake_crc_device(monkeypatch) as (engine, lib):
        reader = _reader(tmp_path / "ck", load_on_engine=True, verify=True)
        out = {k: fake_cuda(torch.zeros_like(v)) for k, v in sd.items() if isinstance(v, torch.Tensor)}
        out["meta"] = {"lr": 0.0, "names": []}
        out["ids"] = torch.zeros_like(sd["ids"])  # a CPU target
        out["w"] = fake_cuda(torch.zeros(64, 96, dtype=torch.float64))  # dtype the engine does not convert
        with pytest.warns(UserWarning, match="without a checksum check"):
            dcp.load(out, storage_reader=reader)
        stats = engine.last_box_load
    n_bytes_io = reader.last_verify["unverified"]
    assert n_bytes_io in (1, 2)  # "meta" as one item or as "meta.lr" + "meta.names"
    assert reader.last_verify["host_records"] == 2 and reader.last_verify["gpu_records"] == stats["verified_records"] == N_RECORDS - 2
    assert out["meta"] == sd["meta"]
    assert torch.equal(plain(out["w"]), sd["w"].double()) and torch.equal(out["ids"], sd["ids"])
    for k in ("b", "flags", "step", "t"):
        assert _bits_equal(out[k], sd[k]), k


def _flip(path, fqn, at=5):
    f, rec = _record(path)[fqn]
    fd = os.open(f, os.O_RDWR)
    try:
        b = os.pread(fd, 1, rec.data_off + at)
        os.pwrite(fd, bytes([b[0] ^ 0x10]), rec.data_off + at)
    finally:
        os.close(fd)


@pytest.mark.parametrize("where", ["engine", "host"])
def test_flipped_byte_raises_before_commit(tmp_path, built_library, monkeypatch, where):
    from torch.distributed.checkpoint.default_planner import DefaultLoadPlanner

    from torch.distributed.checkpoint.api import CheckpointException

    sd = _state()
    dcp.save(sd, checkpoint_id=str(tmp_path / "ck"))
    shutil.copytree(tmp_path / "ck", tmp_path / "bad")
    _flip(tmp_path / "bad", "ids", at=123)
    committed = []
    real = DefaultLoadPlanner.commit_tensor
    monkeypatch.setattr(DefaultLoadPlanner, "commit_tensor", lambda self, req, t: (committed.append(req.dest_index.fqn), real(self, req, t)))
    with fake_crc_device(monkeypatch) as (engine, lib):
        reader = _reader(tmp_path / "bad", load_on_engine=True, verify=True)
        out = _targets(sd)
        if where == "host":
            out["ids"] = torch.zeros_like(sd["ids"])  # the corrupt item takes the stock path
        with pytest.raises(CheckpointException, match=r"(?s)SnapError: .*crc32 mismatch on .*ids in .*__0_0\.distcp at record offset"):
            dcp.load(out, storage_reader=reader)
        assert ("crcx" in lib.calls) == (where == "engine")
    assert committed == []
    # the intact copy loads
    got, stats, _, _ = _verified_load(tmp_path / "ck", sd, monkeypatch)
    assert torch.equal(plain(got["ids"]), sd["ids"])


def test_flipped_byte_without_engine_raises_on_the_host(tmp_path, built_library):
    from torch.distributed.checkpoint.api import CheckpointException

    sd = _state()
    dcp.save(sd, checkpoint_id=str(tmp_path / "ck"))
    _flip(tmp_path / "ck", "w")
    out = {k: torch.zeros_like(v) for k, v in sd.items()}
    with pytest.raises(CheckpointException, match="(?s)SnapError: .*crc32 mismatch on w in"):
        dcp.load(out, storage_reader=_reader(tmp_path / "ck", verify=True))
    reader = _reader(tmp_path / "ck")  # the default does not check
    dcp.load(out, storage_reader=reader)


def test_checkpoint_without_checksums_loads_unverified_and_warns(tmp_path, built_library, monkeypatch):
    sd = _state()
    torch.serialization.set_crc32_options(False)
    try:
        dcp.save(sd, checkpoint_id=str(tmp_path / "ck"))
    finally:
        torch.serialization.set_crc32_options(True)
    assert _record(tmp_path / "ck")["w"][1].crc32 == 0
    ref = _stock(tmp_path / "ck", sd)
    with fake_crc_device(monkeypatch) as (engine, lib):
        reader = _reader(tmp_path / "ck", load_on_engine=True, verify=True)
        out = _targets(sd)
        out["ids"] = torch.zeros_like(sd["ids"])  # and one on the host
        with pytest.warns(UserWarning, match=f"{N_RECORDS} checkpoint items were loaded without a checksum check"):
            dcp.load(out, storage_reader=reader)
        stats = engine.last_box_load
        assert "crcx" not in lib.calls
    assert stats["verified_records"] == 0 and stats["unverified_records"] == N_RECORDS - 1 and stats["verify_extra_bytes"] == 0
    assert reader.last_verify == {"gpu_records": 0, "host_records": 0, "unverified": N_RECORDS}
    for k in sd:
        assert _bits_equal(out[k], ref[k]), k


def test_verify_false_makes_no_checksum_calls(tmp_path, built_library, monkeypatch):
    sd = _state()
    dcp.save(sd, checkpoint_id=str(tmp_path / "ck"))
    with fake_crc_device(monkeypatch) as (engine, lib):
        reader = _reader(tmp_path / "ck", load_on_engine=True)
        before = engine.launches
        out = _targets(sd)
        dcp.load(out, storage_reader=reader)
        stats = engine.last_box_load
        assert lib.calls == ["fill_from_fd", "box_scatter"] and engine.launches - before == 1
        assert set(stats) == {"batches", "peak_staging_bytes", "algorithmic_bytes", "box_ms"}
        # the same load verified adds exactly the checksum launches of its one batch
        before = engine.launches
        lib.calls.clear()
        dcp.load(_targets(sd), storage_reader=_reader(tmp_path / "ck", load_on_engine=True, verify=True))
        assert lib.calls == ["fill_from_fd", "box_scatter", "crcx"] and engine.launches - before == 1 + 2
    assert reader.last_verify is None


def _flip_pickle(path, fqn):
    """Flip one byte inside the ``data.pkl`` of item ``fqn``'s archive (it holds the storage offset, size and stride)."""
    import zipfile

    from nvidia_resiliency_ext.checkpointing.b200.ptzip import _FileWindow

    md = dcp.FileSystemReader(str(path)).read_metadata()
    item = next(v for k, v in md.storage_data.items() if k.fqn == fqn)
    f = os.path.join(str(path), item.relative_path)
    fd = os.open(f, os.O_RDWR)
    try:
        with zipfile.ZipFile(_FileWindow(fd, item.offset, item.length)) as zf:
            pkl = next(i for i in zf.infolist() if i.filename.endswith("/data.pkl"))
        hdr = os.pread(fd, 30, item.offset + pkl.header_offset)
        at = item.offset + pkl.header_offset + 30 + int.from_bytes(hdr[26:28], "little") + int.from_bytes(hdr[28:30], "little")
        at += pkl.file_size // 2
        os.pwrite(fd, bytes([os.pread(fd, 1, at)[0] ^ 0x04]), at)
    finally:
        os.close(fd)
    return f, item


@pytest.mark.parametrize("where", ["engine", "host"])
def test_flipped_byte_in_data_pkl_raises(tmp_path, built_library, monkeypatch, where):
    from torch.distributed.checkpoint.api import CheckpointException
    from torch.distributed.checkpoint.default_planner import DefaultLoadPlanner

    from nvidia_resiliency_ext.checkpointing.b200.ptzip import RecordChecksumError, read_tensor_record

    sd = _state()
    dcp.save(sd, checkpoint_id=str(tmp_path / "ck"))
    f, item = _flip_pickle(tmp_path / "ck", "w")
    fd = os.open(f, os.O_RDONLY)
    try:  # as zipfile reports it (the error before the pickle was read without zipfile)
        with pytest.raises(RecordChecksumError, match=r"not a single-tensor torch.save archive: Bad CRC-32 for file '.*data.pkl'"):
            read_tensor_record(fd, item.offset, item.length)
    finally:
        os.close(fd)
    committed = []
    real = DefaultLoadPlanner.commit_tensor
    monkeypatch.setattr(DefaultLoadPlanner, "commit_tensor", lambda self, req, t: (committed.append(req.dest_index.fqn), real(self, req, t)))
    with fake_crc_device(monkeypatch) as (engine, lib):
        out = _targets(sd)
        if where == "host":
            out["w"] = torch.zeros_like(sd["w"])  # the corrupt item takes the stock path
        with pytest.raises(CheckpointException, match=r"(?s)SnapError: .*crc32 mismatch on w in .*data\.pkl"):
            dcp.load(out, storage_reader=_reader(tmp_path / "ck", load_on_engine=True, verify=True))
        assert committed == []
        # without verify the engine path still refuses the archive, as it did before
        if where == "engine":
            with pytest.raises(CheckpointException, match="Bad CRC-32 for file"):
                dcp.load(_targets(sd), storage_reader=_reader(tmp_path / "ck", load_on_engine=True))
