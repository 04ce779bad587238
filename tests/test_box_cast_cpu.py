"""Converting box scatter without a GPU: fp32 / bf16 / fp16 checkpoints loaded into targets of another of the three dtypes.

The real planner (``nvrx_boxplan_create_cast``) is replayed tile by tile with the numpy conversion oracle, and
``CachedMetadataFileSystemReader(load_on_engine=True)`` runs through a converting variant of the fake box device against the
stock ``FileSystemReader`` (NaN positions compared with isnan, every other element by bits)."""
import contextlib
import ctypes as C
import types

import numpy as np
import pytest
import torch
import torch.distributed.checkpoint as dcp

from _box_oracle import _random_boxes, _random_strides, box_copy
from _cast_oracle import CAST_DTYPES, CAST_OF, PAIRS, SIZE, convert_bytes, special_tensor, tensors_nan_aware_equal
from _fake_box import fake_box_device, fake_cuda
from _fake_device import _val, plain
from _mp import run_ranks

_PAIR_IDS = [f"{str(a)[6:]}-{str(b)[6:]}" for a, b in PAIRS]


# ---------------------------------------------------------------------------------------------------------------------
# planner
# ---------------------------------------------------------------------------------------------------------------------
def _create(boxes, casts, staging_bytes, tile_bytes=0):
    """nvrx_boxplan_create_cast called directly (``casts`` may be None: the NULL pointer); returns (status, handle)."""
    from nvidia_resiliency_ext.checkpointing.b200 import _cabi

    lib = _cabi.lib()
    n = len(boxes)
    flat = lambda k: [int(v) for b in boxes for v in b[k]]  # noqa: E731
    i64 = lambda vals: (C.c_int64 * max(len(vals), 1))(*vals)  # noqa: E731
    h = C.c_void_p()
    rc = lib.nvrx_boxplan_create_cast(
        n, (C.c_uint32 * max(n, 1))(*[b[0] for b in boxes]), (C.c_int32 * max(n, 1))(*[len(b[1]) for b in boxes]),
        i64(flat(1)), (C.c_uint64 * max(n, 1))(*[b[2] for b in boxes]), i64(flat(3)),
        (C.c_void_p * max(n, 1))(*[b[4] or None for b in boxes]), i64(flat(5)),
        None if casts is None else (C.c_uint32 * max(n, 1))(*casts), staging_bytes, tile_bytes, 0, C.byref(h),
    )
    return rc, h


def _plan_view(h, n_boxes):
    """(tiles, per-box geometry + (cast, dst elem)) of a plan handle, through the introspection calls."""
    from nvidia_resiliency_ext.checkpointing.b200 import _cabi

    lib = _cabi.lib()
    nt = C.c_uint64()
    assert lib.nvrx_boxplan_tiles(h, C.byref(nt), None, None, None, None, None, 0) == 0
    cnt = max(nt.value, 1)
    box, nby = (C.c_uint32 * cnt)(), (C.c_uint32 * cnt)()
    row, nrows, off = (C.c_uint64 * cnt)(), (C.c_uint64 * cnt)(), (C.c_uint64 * cnt)()
    assert lib.nvrx_boxplan_tiles(h, None, box, row, nrows, off, nby, nt.value) == 0
    tiles = [(box[i], row[i], nrows[i], off[i], nby[i]) for i in range(nt.value)]
    geo = []
    for b in range(n_boxes):
        rb, no, so, dst = C.c_uint64(), C.c_uint32(), C.c_uint64(), C.c_uint64()
        sz, ss, ds = (C.c_uint64 * 8)(), (C.c_int64 * 8)(), (C.c_int64 * 8)()
        assert lib.nvrx_boxplan_box(h, b, C.byref(rb), C.byref(no), sz, ss, ds, C.byref(so), C.byref(dst)) == 0
        cast, ed = C.c_uint32(), C.c_uint32()
        assert lib.nvrx_boxplan_box_cast(h, b, C.byref(cast), C.byref(ed)) == 0
        k = no.value
        geo.append((rb.value, list(sz)[:k], list(ss)[:k], list(ds)[:k], so.value, dst.value, cast.value, ed.value))
    return tiles, geo


def _destroy(h):
    from nvidia_resiliency_ext.checkpointing.b200 import _cabi

    _cabi.lib().nvrx_boxplan_destroy(h)


def _random_cast_boxes(rng, n_boxes, dst_base):
    """Random boxes (0-8 dims, padded / transposed strides on both sides), about half of them converting; offsets aligned
    to the element sizes.  Returns (boxes as BoxPlan takes them, casts, expected (es, ed, sizes, so, sst, do, dstr, source
    extent bytes), source bytes, destination bytes)."""
    boxes, casts, expect, cur_src, cur_dst = [], [], [], 0, 0
    for _ in range(n_boxes):
        nd = int(rng.integers(0, 9))
        sizes = [int(rng.integers(0 if rng.random() < 0.05 else 1, 5)) for _ in range(nd)]
        while np.prod(sizes, dtype=np.int64) > 3000:
            sizes[int(np.argmax(sizes))] -= 1
        if rng.random() < 0.6:
            code = int(rng.integers(1, 7))
            es, ed = SIZE[CAST_DTYPES[code][0]], SIZE[CAST_DTYPES[code][1]]
        else:
            code, es = 0, int(rng.choice([1, 2, 4, 8, 16]))
            ed = es
        sst, s_ext = _random_strides(rng, sizes)
        dstr, d_ext = _random_strides(rng, sizes)
        src_off = -(-cur_src // es) * es + es * int(rng.integers(0, 10))
        dst_off = -(-cur_dst // 16) * 16 + ed * int(rng.integers(0, 10))
        boxes.append((es, sizes, src_off, sst, dst_base + dst_off, dstr))
        casts.append(code)
        expect.append((es, ed, sizes, src_off, sst, dst_off, dstr, s_ext * es))
        cur_src = src_off + s_ext * es
        cur_dst = dst_off + d_ext * ed
    return boxes, casts, expect, cur_src, cur_dst


def _convert(code, data: np.ndarray) -> np.ndarray:
    return np.frombuffer(convert_bytes(code, data.tobytes()), dtype=np.uint8) if code else data


def _box_expected(src, want, mask, es, ed, code, sizes, so, sst, do, dstr):
    """numpy restatement: gather the box's source elements, convert, scatter them into ``want`` (and count into ``mask``)."""
    if any(s == 0 for s in sizes):
        return
    n = int(np.prod(sizes, dtype=np.int64))
    contig = [0] * len(sizes)
    acc = 1
    for d in range(len(sizes) - 1, -1, -1):
        contig[d] = acc
        acc *= sizes[d]
    packed = np.zeros(n * es, dtype=np.uint8)
    box_copy(src, packed, es, sizes, so, sst, 0, contig)
    box_copy(_convert(code, packed), want, ed, sizes, 0, contig, do, dstr)
    hit = np.zeros(mask.size, dtype=np.uint8)
    box_copy(np.ones(n * ed, dtype=np.uint8), hit, ed, sizes, 0, contig, do, dstr)
    mask += hit


@pytest.mark.parametrize("tile_bytes", [4096, 0])
@pytest.mark.parametrize("seed", range(12))
def test_cast_planner_replay_matches_oracle(built_library, seed, tile_bytes):
    rng = np.random.default_rng(100 + seed)
    dst = np.full(1 << 20, 0xEE, dtype=np.uint8)
    base = dst.ctypes.data
    boxes, casts, expect, src_bytes, dst_bytes = _random_cast_boxes(rng, int(rng.integers(1, 9)), base)
    assert dst_bytes <= dst.size
    # finite source values for the converting boxes' element sizes: random bits of every size, NaN-free enough not to matter
    src = rng.integers(0, 256, src_bytes + 1, dtype=np.uint8)
    rc, h = _create(boxes, casts, src_bytes, tile_bytes)
    assert rc == 0
    try:
        tiles, geo = _plan_view(h, len(boxes))
        # copy tiles first, then converting tiles
        kinds = [bool(casts[t[0]]) for t in tiles]
        assert kinds == sorted(kinds)
        written = np.zeros(dst.size, dtype=np.int32)
        got = dst.copy()
        for b, row, nrows, off, nby in tiles:
            rb, sz, ss, ds, so, dbase, code, ed = geo[b]
            es = boxes[b][0]
            assert code == casts[b] and ed == expect[b][1]
            assert rb % es == 0 and off % es == 0 and (nrows > 1 or nby % es == 0)
            ext_lo, ext_hi = expect[b][3], expect[b][3] + expect[b][7]
            for r in range(row, row + nrows):
                s, d, q = so, dbase - base, r
                for k in range(len(sz) - 1, -1, -1):
                    q, i = divmod(q, sz[k])
                    s += i * ss[k]
                    d += i * ds[k]
                lo, n = (off, nby) if nrows == 1 else (0, rb)
                assert ext_lo <= s + lo and s + lo + n <= ext_hi <= src_bytes  # source read inside the box's extent
                out = _convert(code, src[s + lo : s + lo + n])
                dlo = d + lo // es * ed
                written[dlo : dlo + out.size] += 1
                got[dlo : dlo + out.size] = out
        want = np.full_like(dst, 0xEE)
        mask = np.zeros(dst.size, dtype=np.int32)
        for (es, ed, sizes, so, sst, do, dstr, _), code in zip(expect, casts):
            _box_expected(src, want, mask, es, ed, code, sizes, so, sst, do, dstr)
        assert np.array_equal(written, mask), "every destination byte exactly once, nothing outside the views"
        assert np.array_equal(got, want)
        info_tiles, algo = C.c_uint64(), C.c_uint64()
        from nvidia_resiliency_ext.checkpointing.b200 import _cabi

        assert _cabi.lib().nvrx_boxplan_info(h, C.byref(info_tiles), C.byref(algo)) == 0
        assert algo.value == sum(int(np.prod(e[2], dtype=np.int64)) * (e[0] + e[1]) for e in expect)
    finally:
        _destroy(h)


@pytest.mark.parametrize("seed", range(8))
def test_cast_null_and_all_zero_reproduce_boxplan_create(built_library, seed):
    from nvidia_resiliency_ext.checkpointing.b200.engine import BoxPlan

    rng = np.random.default_rng(seed)
    dst = np.zeros(1 << 20, dtype=np.uint8)
    boxes, _, src_bytes, _ = _random_boxes(rng, int(rng.integers(1, 8)), dst.ctypes.data)
    for tile in (4096, 0):
        ref = BoxPlan(boxes, src_bytes, device=0, tile_bytes=tile)
        want = _plan_view(ref._h, len(boxes))
        for casts in (None, [0] * len(boxes)):
            rc, h = _create(boxes, casts, src_bytes, tile)
            assert rc == 0
            try:
                assert _plan_view(h, len(boxes)) == want
            finally:
                _destroy(h)
        ref.close()


def test_cast_planner_rejects_malformed_input(built_library):
    from nvidia_resiliency_ext.checkpointing.b200 import _cabi

    buf = np.zeros(256, dtype=np.uint8)
    p = (buf.ctypes.data + 15) // 16 * 16
    bad = [
        ([(4, [4], 0, [1], p, [1])], [7]),  # unknown code
        ([(4, [4], 0, [1], p, [1])], [0xFFFFFFFF]),
        ([(2, [4], 0, [1], p, [1])], [1]),  # fp32 -> bf16 with a 2-byte source element
        ([(4, [4], 0, [1], p, [1])], [3]),  # bf16 -> fp32 with a 4-byte source element
        ([(4, [4], 0, [1], p, [1])], [6]),
        ([(4, [4], 2, [1], p, [1])], [1]),  # source offset not a multiple of 4
        ([(2, [4], 1, [1], p, [1])], [5]),  # ... of 2
        ([(2, [4], 0, [1], p + 2, [1])], [3]),  # destination not 4-byte aligned for fp32
        ([(4, [4], 0, [1], p + 1, [1])], [2]),  # ... not 2-byte aligned for fp16
        ([(4, [4], 4, [1], p, [1])], [1]),  # last source byte beyond staging (16 bytes)
    ]
    for boxes, casts in bad:
        rc, h = _create(boxes, casts, 16)
        assert rc == _cabi.E_INVALID, (boxes, casts)
    rc, h = _create([(4, [4], 0, [1], p, [1]), (2, [2, 3], 16, [3, 1], p + 64, [1, 2]), (2, [0], 0, [1], 0, [1])], [1, 4, 5], 32)
    assert rc == 0
    tiles, geo = _plan_view(h, 3)
    assert [g[6:] for g in geo] == [(1, 2), (4, 4), (5, 2)]
    assert geo[0][0] == 16  # row_bytes in source bytes
    _destroy(h)


def test_wide_destination_tiles_count_source_bytes(built_library):
    """A long bf16 -> fp32 run: tiles are cut so the wider (destination) side stays at tile_bytes."""
    buf = np.zeros(1 << 20, dtype=np.uint8)
    p = (buf.ctypes.data + 15) // 16 * 16
    rc, h = _create([(2, [100000], 0, [1], p, [1]), (4, [100000], 0, [1], p, [1])], [3, 1], 400000, 4096)
    assert rc == 0
    tiles, geo = _plan_view(h, 2)
    assert all(t[4] == 2048 for t in tiles if t[0] == 0 and t[3] + 2048 < 200000)  # 2048 source -> 4096 destination bytes
    assert all(t[4] == 4096 for t in tiles if t[0] == 1 and t[3] + 4096 < 400000)
    assert sum(t[4] for t in tiles if t[0] == 0) == 200000 and sum(t[4] for t in tiles if t[0] == 1) == 400000
    _destroy(h)


# ---------------------------------------------------------------------------------------------------------------------
# the converting fake device
# ---------------------------------------------------------------------------------------------------------------------
def _box_scatter_cast(self, h, staging, stream):
    """The real planner's tiles replayed on host memory: bit copies with memmove, conversions with the numpy oracle."""
    n = C.c_uint64()
    assert self._real.nvrx_boxplan_tiles(h, C.byref(n), None, None, None, None, None, 0) == 0
    cnt = max(n.value, 1)
    box, nby = (C.c_uint32 * cnt)(), (C.c_uint32 * cnt)()
    row, nrows, off = (C.c_uint64 * cnt)(), (C.c_uint64 * cnt)(), (C.c_uint64 * cnt)()
    assert self._real.nvrx_boxplan_tiles(h, None, box, row, nrows, off, nby, n.value) == 0
    geo, kernels = {}, set()
    for t in range(n.value):
        b = box[t]
        if b not in geo:
            rb, no, so, dst = C.c_uint64(), C.c_uint32(), C.c_uint64(), C.c_uint64()
            sz, ss, ds = (C.c_uint64 * 8)(), (C.c_int64 * 8)(), (C.c_int64 * 8)()
            assert self._real.nvrx_boxplan_box(h, b, C.byref(rb), C.byref(no), sz, ss, ds, C.byref(so), C.byref(dst)) == 0
            code, ed = C.c_uint32(), C.c_uint32()
            assert self._real.nvrx_boxplan_box_cast(h, b, C.byref(code), C.byref(ed)) == 0
            k = no.value
            es = SIZE[CAST_DTYPES[code.value][0]] if code.value else ed.value
            geo[b] = (rb.value, list(sz)[:k], list(ss)[:k], list(ds)[:k], so.value, dst.value, code.value, es, ed.value)
        rb, sz, ss, ds, so, dst, code, es, ed = geo[b]
        kernels.add("box_scatter_cast" if code else "box_scatter")
        for r in range(row[t], row[t] + nrows[t]):
            s_addr, d_addr, q = _val(staging) + so, dst, r
            for d in range(len(sz) - 1, -1, -1):
                q, i = divmod(q, sz[d])
                s_addr += i * ss[d]
                d_addr += i * ds[d]
            lo, length = (off[t], nby[t]) if nrows[t] == 1 else (0, rb)
            if code:
                out = convert_bytes(code, C.string_at(s_addr + lo, length))
                C.memmove(d_addr + lo // es * ed, out, len(out))
            else:
                C.memmove(d_addr + lo, s_addr + lo, length)
    self.calls.extend(k for k in ("box_scatter", "box_scatter_cast") if k in kernels)
    return 0


@contextlib.contextmanager
def fake_cast_box_device(monkeypatch):
    """``fake_box_device`` whose box scatter also converts; counts ``nvrx_boxplan_create_cast`` calls in ``lib.creates``."""
    with fake_box_device(monkeypatch) as (engine, lib):
        lib.nvrx_box_scatter = types.MethodType(_box_scatter_cast, lib)
        lib.creates = {"plain": 0, "cast": 0}
        real_create, real_cast = lib._real.nvrx_boxplan_create, lib._real.nvrx_boxplan_create_cast

        def create(*a):
            lib.creates["plain"] += 1
            return real_create(*a)

        def create_cast(*a):
            lib.creates["cast"] += 1
            return real_cast(*a)

        lib.nvrx_boxplan_create = create
        lib.nvrx_boxplan_create_cast = create_cast
        yield engine, lib


# ---------------------------------------------------------------------------------------------------------------------
# reader through the converting fake device
# ---------------------------------------------------------------------------------------------------------------------
def _state(dtype, seed=0):
    g = torch.Generator().manual_seed(seed)
    w = torch.randn(64, 96, generator=g) * 3
    sp = special_tensor(dtype)
    w = w.to(dtype)
    w.view(-1)[5 : 5 + sp.numel()] = sp
    w.view(-1)[3001 : 3001 + sp.numel()] = sp
    return {
        "w": w,
        "b": torch.randn(97, generator=g).to(dtype),
        "odd": torch.randn(5, 7, 3, generator=g).to(dtype),
        "step": torch.tensor(7.25).to(dtype),
        "empty": torch.empty(0, 5, dtype=dtype),
        "t": torch.randn(24, 40, generator=g).t().to(dtype),  # saved with transposed strides
    }


def _stock(path, like, dtype):
    out = {k: torch.zeros(v.shape, dtype=dtype) for k, v in like.items()}
    dcp.load(out, storage_reader=dcp.FileSystemReader(str(path)))
    return out


def _engine_load(path, like, dtype, *, contiguous=True):
    from nvidia_resiliency_ext.checkpointing.async_ckpt.cached_metadata_filesystem_reader import CachedMetadataFileSystemReader

    out = {}
    for k, v in like.items():
        if contiguous or v.dim() != 2:
            out[k] = fake_cuda(torch.full(v.shape, 3, dtype=dtype))
        else:
            out[k] = fake_cuda(torch.full((v.shape[1], v.shape[0]), 3, dtype=dtype)).t()  # transposed target view
    CachedMetadataFileSystemReader.clear_metadata_cache()
    dcp.load(out, storage_reader=CachedMetadataFileSystemReader(str(path), load_on_engine=True))
    return out


def _assert_same(got, ref):
    for k in ref:
        assert tensors_nan_aware_equal(plain(got[k]), ref[k]), k


@pytest.mark.parametrize("contiguous", [True, False])
@pytest.mark.parametrize("pair", PAIRS, ids=_PAIR_IDS)
def test_reader_cast_same_layout_matches_stock(tmp_path, built_library, monkeypatch, pair, contiguous):
    src, dst = pair
    sd = _state(src)
    dcp.save(sd, checkpoint_id=str(tmp_path / "ck"))
    ref = _stock(tmp_path / "ck", sd, dst)
    with fake_cast_box_device(monkeypatch) as (engine, lib):
        got = _engine_load(tmp_path / "ck", sd, dst, contiguous=contiguous)
        assert lib.calls.count("box_scatter_cast") == 1 and "box_scatter" not in lib.calls and engine.box_loads == 1
        assert lib.creates == {"plain": 0, "cast": 1}
        stats = engine.last_box_load
    n = sum(v.numel() for v in sd.values())
    assert stats["algorithmic_bytes"] == n * (SIZE[src] + SIZE[dst])
    _assert_same(got, ref)


def _save_sharded(rank, world, root, placement, dtype):
    from torch.distributed.device_mesh import init_device_mesh
    from torch.distributed.tensor import Shard, distribute_tensor

    mesh = init_device_mesh("cpu", (world,))
    sd = {k: distribute_tensor(v.contiguous(), mesh, [Shard(placement if v.dim() > placement else 0)])
          for k, v in _state(dtype).items() if v.dim() >= 1 and v.numel()}
    dcp.save(sd, checkpoint_id=root)


@pytest.mark.parametrize("placement", [0, 1])
@pytest.mark.parametrize("pair", PAIRS, ids=_PAIR_IDS)
def test_reader_cast_two_rank_shards_match_stock(tmp_path, built_library, monkeypatch, pair, placement):
    src, dst = pair
    root = str(tmp_path / f"shard{placement}")
    run_ranks(_save_sharded, 2, root, placement, src)
    full = {k: v.contiguous() for k, v in _state(src).items() if v.dim() >= 1 and v.numel()}
    ref = _stock(root, full, dst)
    with fake_cast_box_device(monkeypatch) as (engine, lib):
        got = _engine_load(root, full, dst, contiguous=False)
        assert "box_scatter_cast" in lib.calls
    _assert_same(got, ref)


@pytest.mark.parametrize("pair", PAIRS, ids=_PAIR_IDS)
def test_reader_cast_budget_smaller_than_one_item(tmp_path, built_library, monkeypatch, pair):
    from nvidia_resiliency_ext.checkpointing.b200.engine import SnapshotEngine

    src, dst = pair
    sd = _state(src)
    dcp.save(sd, checkpoint_id=str(tmp_path / "ck"))
    ref = _stock(tmp_path / "ck", sd, dst)
    monkeypatch.setattr(SnapshotEngine, "DCP_LOAD_STAGING", 4096)
    with fake_cast_box_device(monkeypatch) as (engine, lib):
        got = _engine_load(tmp_path / "ck", sd, dst, contiguous=False)
        stats = engine.last_box_load
    assert stats["batches"] > 3 and stats["peak_staging_bytes"] <= 4096
    _assert_same(got, ref)


def _mixed_state():
    g = torch.Generator().manual_seed(3)
    return {
        "f32": torch.randn(33, 20, generator=g),
        "bf16": torch.randn(40, generator=g).to(torch.bfloat16),
        "f16": torch.randn(7, 9, generator=g).to(torch.float16),
        "f32_to_f64": torch.randn(6, 5, generator=g),
        "ids": torch.randint(0, 1 << 30, (33, 7), generator=g),
        "ids_cpu": torch.randint(0, 1 << 20, (9,), generator=g),
        "c": torch.randn(9, 4, dtype=torch.complex64, generator=g),
        "flags": torch.rand(17, 5, generator=g) > 0.5,
        "f16_cpu": torch.randn(8, generator=g).to(torch.float16),
        "same": torch.randn(11, 3, generator=g),
    }


def test_reader_cast_routing(tmp_path, built_library, monkeypatch):
    from nvidia_resiliency_ext.checkpointing.async_ckpt.cached_metadata_filesystem_reader import CachedMetadataFileSystemReader

    sd = _mixed_state()
    sd["meta"] = {"lr": 0.1}  # BYTE_IO
    dcp.save(sd, checkpoint_id=str(tmp_path / "ck"))
    seen = []
    real = dcp.FileSystemReader.read_data

    def spy(self, plan, planner):
        seen.extend(item.dest_index.fqn for item in plan.items)
        return real(self, plan, planner)

    monkeypatch.setattr(dcp.FileSystemReader, "read_data", spy)
    targets = {
        "f32": torch.bfloat16, "bf16": torch.float16, "f16": torch.float32, "f32_to_f64": torch.float64,
        "ids": torch.int32, "c": torch.complex128, "flags": torch.uint8, "same": torch.float32,
    }
    with fake_cast_box_device(monkeypatch) as (engine, lib):
        out = {k: fake_cuda(torch.zeros(sd[k].shape, dtype=dt)) for k, dt in targets.items()}
        out["ids_cpu"] = torch.zeros(9, dtype=torch.int32)  # CPU targets, with and without a float conversion
        out["f16_cpu"] = torch.zeros(8, dtype=torch.bfloat16)
        out["meta"] = {"lr": 0.0}
        CachedMetadataFileSystemReader.clear_metadata_cache()
        dcp.load(out, storage_reader=CachedMetadataFileSystemReader(str(tmp_path / "ck"), load_on_engine=True))
        assert lib.calls.count("box_scatter") == 1 and lib.calls.count("box_scatter_cast") == 1
    assert sorted(set(seen)) in (
        ["c", "f16_cpu", "f32_to_f64", "flags", "ids", "ids_cpu", "meta.lr"],
        ["c", "f16_cpu", "f32_to_f64", "flags", "ids", "ids_cpu", "meta"],
    )
    assert out["meta"] == sd["meta"]
    for k, v in out.items():
        if k != "meta":
            assert tensors_nan_aware_equal(plain(v), sd[k].to(v.dtype)), k


def _record_plans(monkeypatch):
    """Replace engine.BoxPlan by a subclass that records every (boxes, casts) it is built with."""
    from nvidia_resiliency_ext.checkpointing.b200 import engine as eng

    made = []

    class Recording(eng.BoxPlan):
        def __init__(self, boxes, staging_bytes, **kw):
            made.append((list(boxes), kw.get("casts")))
            super().__init__(boxes, staging_bytes, **kw)

    monkeypatch.setattr(eng, "BoxPlan", Recording)
    return made


def test_copy_piece_positions_unchanged_without_casts(tmp_path, built_library, monkeypatch):
    """A checkpoint without conversions: every piece at the first position >= the cursor congruent to its target mod 16,
    planned by nvrx_boxplan_create."""
    from nvidia_resiliency_ext.checkpointing.b200.engine import box_span

    from nvidia_resiliency_ext.checkpointing.async_ckpt.cached_metadata_filesystem_reader import CachedMetadataFileSystemReader

    sd = _state(torch.float32)
    sd["h"] = torch.randn(13, 5).to(torch.float16)
    dcp.save(sd, checkpoint_id=str(tmp_path / "ck"))
    made = _record_plans(monkeypatch)
    with fake_cast_box_device(monkeypatch) as (engine, lib):
        out = {k: fake_cuda(torch.zeros(v.shape, dtype=v.dtype)) for k, v in sd.items()}
        CachedMetadataFileSystemReader.clear_metadata_cache()
        dcp.load(out, storage_reader=CachedMetadataFileSystemReader(str(tmp_path / "ck"), load_on_engine=True))
        assert lib.creates == {"plain": 1, "cast": 0}
    assert len(made) == 1
    boxes, casts = made[0]
    assert not any(casts)
    cur = 0
    for es, sizes, pos, sst, dst, dstr in boxes:
        assert pos == cur + (dst - cur) % 16
        cur = pos + box_span(sizes, sst, es)


@pytest.mark.parametrize("pair", PAIRS, ids=_PAIR_IDS)
def test_cast_piece_positions_follow_the_placement_rule(tmp_path, built_library, monkeypatch, pair):
    from nvidia_resiliency_ext.checkpointing.b200.engine import box_span

    from nvidia_resiliency_ext.checkpointing.b200.engine import SnapshotEngine

    src, dst_dtype = pair
    sd = _state(src)
    dcp.save(sd, checkpoint_id=str(tmp_path / "ck"))
    made = _record_plans(monkeypatch)
    monkeypatch.setattr(SnapshotEngine, "DCP_LOAD_STAGING", 4096)  # several batches: positions restart at 0
    with fake_cast_box_device(monkeypatch) as (engine, lib):
        got = _engine_load(tmp_path / "ck", sd, dst_dtype, contiguous=False)
    v = 4 if torch.float32 in pair else 8
    es, ed = SIZE[src], SIZE[dst_dtype]
    n_cast = 0
    for boxes, casts in made:
        cur = 0
        for (e, sizes, pos, sst, dst, dstr), code in zip(boxes, casts):
            assert code == CAST_OF[pair] and e == es
            assert pos >= cur and pos - cur < 16
            assert pos % es == 0 and (pos // es) % v == (dst // ed) % v
            cur = pos + box_span(sizes, sst, es)
            n_cast += 1
    assert len(made) > 1 and n_cast > len(sd)  # every non-empty item, several pieces for "w"
    _assert_same(got, _stock(tmp_path / "ck", sd, dst_dtype))
