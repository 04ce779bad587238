"""GPU tests of the converting box scatter: fp32 / bf16 / fp16 checkpoint items loaded into targets of another of the three.

ABI level (``nvrx_box_scatter`` of ``nvrx_boxplan_create_cast`` plans): destinations are filled with a sentinel first and
every byte of the buffer, guard included, is compared with the numpy oracle (tests/_cast_oracle.py); staging must be left
unchanged.  Source values there are finite (bit 14 of every 16-bit word cleared), so the comparison is bit-exact; the
special-values test covers NaN (compared with isnan), inf, subnormals, ties and overflow.  End to end, the engine reader must
match the stock ``FileSystemReader`` element by element (NaN positions by isnan, everything else by bits)."""
import numpy as np
import pytest
import torch
import torch.distributed.checkpoint as dcp
from torch.distributed.checkpoint import DefaultSavePlanner, FileSystemReader

from _box_oracle import _contig_strides, box_copy
from _cast_oracle import (
    CAST_DTYPES,
    CAST_OF,
    PAIRS,
    SIZE,
    UINT,
    convert_bits,
    convert_bytes,
    nan_aware_equal,
    special_tensor,
    tensor_bits,
    tensors_nan_aware_equal,
)
from _mp import run_ranks

pytestmark = pytest.mark.gpu

SENTINEL = 0xA5
GUARD = 512
_PAIR_IDS = [f"{str(a)[6:]}-{str(b)[6:]}" for a, b in PAIRS]


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _round(v, a):
    return -(-v // a) * a


def _finite_bytes(rng, n):
    """Random bytes in which every aligned 16-bit word, read as fp16 or bf16 (and every 32-bit word as fp32), is finite."""
    raw = rng.integers(0, 256, _round(n, 4), dtype=np.uint8)
    raw.view(np.uint16)[:] &= 0xBFFF
    return raw[:n].copy()


def _assert_bytes(got, want, what):
    got = got.cpu().numpy() if isinstance(got, torch.Tensor) else got
    assert got.shape == want.shape, what
    bad = np.flatnonzero(got != want)
    assert bad.size == 0, f"{what}: {bad.size} wrong bytes, first at {bad[0]} (got {got[bad[0]]:#x}, want {want[bad[0]]:#x})"


def _expected(src, want, code, es, ed, sizes, so, sst, do, dstr):
    """Gather the box's source elements, convert them with the oracle, scatter them into ``want``."""
    if any(s == 0 for s in sizes):
        return
    n = int(np.prod(sizes, dtype=np.int64))
    contig = _contig_strides(sizes)
    packed = np.zeros(n * es, dtype=np.uint8)
    box_copy(src, packed, es, sizes, so, sst, 0, contig)
    out = np.frombuffer(convert_bytes(code, packed.tobytes()), dtype=np.uint8) if code else packed
    box_copy(out, want, ed, sizes, 0, contig, do, dstr)


def _run(boxes, casts, src, dst_len, tile=0):
    """boxes: (es, sizes, src_off, src_strides, dst_off, dst_strides), offsets in bytes; returns the plan after checking
    every destination byte and the staging bytes."""
    from nvidia_resiliency_ext.checkpointing.b200.engine import BoxPlan

    stg = torch.from_numpy(src).cuda()
    dst = torch.full((dst_len + GUARD,), SENTINEL, dtype=torch.uint8, device="cuda")
    bp = BoxPlan([(es, sz, so, ss, dst.data_ptr() + do, ds) for es, sz, so, ss, do, ds in boxes], src.size,
                 device=torch.cuda.current_device(), tile_bytes=tile, casts=casts)
    bp.scatter(stg.data_ptr(), _stream())
    torch.cuda.synchronize()
    want = np.full(dst.numel(), SENTINEL, dtype=np.uint8)
    for (es, sz, so, ss, do, ds), code in zip(boxes, casts):
        ed = SIZE[CAST_DTYPES[code][1]] if code else es
        _expected(src, want, code, es, ed, sz, so, ss, do, ds)
    _assert_bytes(dst, want, "converting box scatter")
    _assert_bytes(stg, src, "box scatter staging")
    return bp


def _vec(pair):
    return 4 if torch.float32 in pair else 8


# ---------------------------------------------------------------------------------------------------------------------
# ABI level
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("pair", PAIRS, ids=_PAIR_IDS)
def test_runs_of_every_length_at_every_offset(built_library, pair):
    """Runs of 1-70 elements starting at every destination element offset mod 8, with the staging position following the
    placement rule (vector body) and breaking it by one element (element-load fallback)."""
    code, es, ed, v = CAST_OF[pair], SIZE[pair[0]], SIZE[pair[1]], _vec(pair)
    boxes, cs, cd = [], 0, 0
    for placed in (True, False):
        for n in range(1, 71):
            for k in range(8):
                do = _round(cd, 16) + k * ed
                so = _round(cs, 16) + ((k if placed else k + 1) % v) * es
                boxes.append((es, [n], so, [1], do, [1]))
                cs, cd = so + n * es, do + n * ed
    src = _finite_bytes(np.random.default_rng(code), cs)
    bp = _run(boxes, [code] * len(boxes), src, cd)
    assert bp.launches == 1 and all(t[2] == 1 for t in bp.tiles())  # each run: one row, a whole CTA
    bp.close()


def _hand_boxes(es):
    """(sizes, src strides, dst strides) in elements, per tile shape."""
    return [
        ([200_004 // es + 5], [1], [1]),  # a run of > 200 000 source bytes: byte ranges of tiles, a CTA each
        ([300, 40], [43, 1], [41, 1]),  # >= 32-byte rows grouped: a warp per row
        ([300, 3], [5, 1], [4, 1]),  # < 32-byte rows: a thread per row
        ([700, 90], [1, 700], [90, 1]),  # strided innermost dim on the source side: element-wise
        ([50, 60], [60, 1], [1, 50]),  # ... on the destination side
        ([2, 3, 2, 2, 3, 2, 2, 3], _contig_strides([3, 4, 3, 3, 4, 3, 3, 4]), _contig_strides([2, 4, 2, 3, 3, 3, 2, 4])),
        ([5, 1000], [0, 1], [1000, 1]),  # zero-stride source dim: one saved row broadcast into five
    ]


def _extent(sizes, strides, elem):
    return elem * (1 + sum((n - 1) * s for n, s in zip(sizes, strides))) if all(sizes) else 0


@pytest.mark.parametrize("placed", [True, False], ids=["placed", "misplaced"])
@pytest.mark.parametrize("tile", [4096, 32768])
@pytest.mark.parametrize("pair", PAIRS, ids=_PAIR_IDS)
def test_hand_made_geometry(built_library, pair, tile, placed):
    code, es, ed, v = CAST_OF[pair], SIZE[pair[0]], SIZE[pair[1]], _vec(pair)
    boxes, cs, cd = [], 0, 0
    for i, (sizes, sst, dstr) in enumerate(_hand_boxes(es)):
        k = (3 * i + 1) % 8
        do = _round(cd, 16) + k * ed
        so = _round(cs, 16) + ((k if placed else k + 3) % v) * es
        boxes.append((es, sizes, so, sst, do, dstr))
        cs, cd = so + _extent(sizes, sst, es), do + _extent(sizes, dstr, ed)
    src = _finite_bytes(np.random.default_rng(tile + code), cs)
    bp = _run(boxes, [code] * len(boxes), src, cd, tile)
    tiles = bp.tiles()
    assert sum(1 for t in tiles if t[0] == 0) > 1 and all(t[2] == 1 for t in tiles if t[0] == 0)
    assert any(t[2] > 1 for t in tiles if t[0] == 1) and any(t[2] > 1 for t in tiles if t[0] == 2)
    assert all(t[3] % es == 0 and t[4] % es == 0 for t in tiles)
    bp.close()


def _kernel_launches(fn):
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    names = [e.name for e in prof.events() if "walk_box" in e.name]
    return sorted("cast" if "walk_box_cast" in n else "copy" for n in names)


def test_mixed_batch_launches_copy_then_cast(built_library):
    """Copy and converting boxes in one batch: two launches (walk_box, then walk_box_cast); without a cast one."""
    rng = np.random.default_rng(7)
    boxes, casts, cs, cd = [], [], 0, 0
    for i, code in enumerate([0, 1, 0, 3, 5, 0, 2, 4, 6]):
        es = SIZE[CAST_DTYPES[code][0]] if code else (4, 2, 8)[i % 3]
        ed = SIZE[CAST_DTYPES[code][1]] if code else es
        sizes, sst, dstr = [37, 129], [131, 1], [129, 1]
        so, do = _round(cs, 16) + 2 * es * (i % 2), _round(cd, 16) + 2 * ed * (i % 2)
        boxes.append((es, sizes, so, sst, do, dstr))
        casts.append(code)
        cs, cd = so + _extent(sizes, sst, es), do + _extent(sizes, dstr, ed)
    src = _finite_bytes(rng, cs)
    bp = _run(boxes, casts, src, cd, 4096)
    kinds = [bool(casts[t[0]]) for t in bp.tiles()]
    assert kinds == sorted(kinds) and bp.launches == 2
    stg = torch.from_numpy(src).cuda()
    assert _kernel_launches(lambda: bp.scatter(stg.data_ptr(), _stream())) == ["cast", "copy"]
    bp.close()
    plain = [b for b, c in zip(boxes, casts) if not c]
    bp = _run(plain, [0] * len(plain), src, cd, 4096)
    assert bp.launches == 1
    assert _kernel_launches(lambda: bp.scatter(stg.data_ptr(), _stream())) == ["copy"]
    bp.close()
    only = [b for b, c in zip(boxes, casts) if c]
    bp = _run(only, [c for c in casts if c], src, cd, 4096)
    assert _kernel_launches(lambda: bp.scatter(stg.data_ptr(), _stream())) == ["cast"]
    bp.close()


@pytest.mark.parametrize("pair", PAIRS, ids=_PAIR_IDS)
def test_special_values_match_oracle_and_torch(built_library, pair):
    """+-0, +-inf, NaNs of both signs with payloads, fp32 subnormals, values that become bf16 / fp16 subnormals, RNE ties
    both ways, the fp16 overflow edge and fp32 max -> bf16, each at every position mod 8 (vector body, head and tail)."""
    from nvidia_resiliency_ext.checkpointing.b200.engine import BoxPlan

    code, es, ed = CAST_OF[pair], SIZE[pair[0]], SIZE[pair[1]]
    sp = special_tensor(pair[0])
    x = torch.cat([torch.roll(sp, k) for k in range(8)] + [sp[:5]])
    bits = tensor_bits(x)
    stg = x.cuda()
    out = torch.full((x.numel() + 64,), float("nan"), dtype=pair[1], device="cuda")
    out.view(torch.uint8).fill_(SENTINEL)
    bp = BoxPlan([(es, [x.numel()], 0, [1], out.data_ptr(), [1])], x.numel() * es, device=torch.cuda.current_device(),
                 casts=[code])
    bp.scatter(stg.data_ptr(), _stream())
    torch.cuda.synchronize()
    got = tensor_bits(out)
    want = convert_bits(code, bits).astype(UINT[ed])
    assert nan_aware_equal(got[: x.numel()], want, pair[1])
    assert (out.view(torch.uint8)[x.numel() * ed :] == SENTINEL).all()
    assert tensor_bits(stg).tobytes() == bits.tobytes()
    # the oracle is what torch computes on the host, up to NaN bits
    assert nan_aware_equal(tensor_bits(x.to(pair[1])), want, pair[1])
    if pair[0] == torch.float32:
        nan_out = got[: x.numel()][np.isnan(x.numpy())]
        if pair[1] != torch.float32:
            assert (nan_out == 0x7FFF).all()  # the device's canonical NaN
    bp.close()


# ---------------------------------------------------------------------------------------------------------------------
# dcp end to end
# ---------------------------------------------------------------------------------------------------------------------
def _state(dtype, device="cuda"):
    g = torch.Generator().manual_seed(3)
    w = (torch.randn(1000, 768, generator=g) * 4).to(dtype)
    sp = special_tensor(dtype)
    for at in (0, 3, 1001, 400_005):
        w.view(-1)[at : at + sp.numel()] = sp
    sd = {
        "w": w,
        "b": torch.randn(4099, generator=g).to(dtype),
        "odd": torch.randn(5, 7, 3, generator=g).to(dtype),
        "step": torch.tensor(7.0).to(dtype),
        "empty": torch.empty(0, 5, dtype=dtype),
        "t": (torch.randn(384, 640, generator=g) * 1e-3).t().to(dtype),  # saved with transposed strides
    }
    return {k: v.to(device) for k, v in sd.items()}


def _targets(like, dtype, contiguous=True, device="cuda"):
    out = {}
    for k, v in like.items():
        if contiguous or v.dim() != 2:
            out[k] = torch.zeros(v.shape, dtype=dtype, device=device)
        else:
            out[k] = torch.zeros(v.shape[1], v.shape[0], dtype=dtype, device=device).t()
    return out


def _stock(path, like, dtype):
    out = _targets(like, dtype, device="cpu")
    dcp.load(out, storage_reader=FileSystemReader(str(path)))
    return out


def _engine(path, like, dtype, contiguous=True):
    from nvidia_resiliency_ext.checkpointing.async_ckpt.cached_metadata_filesystem_reader import CachedMetadataFileSystemReader

    out = _targets(like, dtype, contiguous)
    CachedMetadataFileSystemReader.clear_metadata_cache()
    dcp.load(out, storage_reader=CachedMetadataFileSystemReader(str(path), load_on_engine=True))
    torch.cuda.synchronize()
    return out


def _assert_same(got, ref):
    for k in ref:
        assert got[k].is_cuda, k
        assert tensors_nan_aware_equal(got[k], ref[k]), k


def _save_sharded(rank, world, root, placement, dtype):
    from torch.distributed.device_mesh import init_device_mesh
    from torch.distributed.tensor import Shard, distribute_tensor

    mesh = init_device_mesh("cpu", (world,))
    sd = {k: distribute_tensor(v.contiguous(), mesh, [Shard(placement if v.dim() > placement else 0)])
          for k, v in _state(dtype, "cpu").items() if v.dim() >= 1 and v.numel()}
    dcp.save(sd, checkpoint_id=root)


@pytest.fixture(scope="module")
def checkpoints(tmp_path_factory):
    """One checkpoint per (saved dtype, layout), written once for the module."""
    made = {}

    def get(dtype, layout):
        key = (dtype, layout)
        if key not in made:
            root = str(tmp_path_factory.mktemp(f"{str(dtype)[6:]}_{layout}"))
            if layout == "same":
                dcp.save(_state(dtype), checkpoint_id=root)
            else:
                run_ranks(_save_sharded, 2, root, int(layout[-1]), dtype)
            made[key] = root
        return made[key]

    return get


@pytest.mark.parametrize("contiguous", [True, False], ids=["contiguous", "transposed"])
@pytest.mark.parametrize("layout", ["same", "shard0", "shard1"])
@pytest.mark.parametrize("pair", PAIRS, ids=_PAIR_IDS)
def test_dcp_load_converts_like_the_stock_reader(built_library, checkpoints, pair, layout, contiguous):
    from nvidia_resiliency_ext.checkpointing.b200.engine import SnapshotEngine

    src, dst = pair
    root = checkpoints(src, layout)
    like = _state(src)
    if layout != "same":
        like = {k: v.contiguous() for k, v in like.items() if v.dim() >= 1 and v.numel()}
    ref = _stock(root, like, dst)
    eng = SnapshotEngine.get()
    before = eng.box_batches
    got = _engine(root, like, dst, contiguous)
    assert eng.box_batches > before
    n = sum(v.numel() for v in like.values())
    assert eng.last_box_load["algorithmic_bytes"] == n * (SIZE[src] + SIZE[dst])
    _assert_same(got, ref)


def test_mixed_plan_with_conversions(tmp_path, built_library):
    from nvidia_resiliency_ext.checkpointing.async_ckpt.cached_metadata_filesystem_reader import CachedMetadataFileSystemReader

    g = torch.Generator().manual_seed(5)
    sd = {
        "f32": torch.randn(300, 77, generator=g).cuda(),
        "bf16": torch.randn(4099, generator=g).to(torch.bfloat16).cuda(),
        "f16": torch.randn(64, 48, generator=g).to(torch.float16).cuda(),
        "f64": torch.randn(30, 7, generator=g).cuda(),
        "ids": torch.randint(0, 1 << 40, (33, 7), generator=g).cuda(),
        "same": torch.randn(129, 3, generator=g).cuda(),
        "meta": {"lr": 0.1},
    }
    dcp.save(sd, checkpoint_id=str(tmp_path / "ck"))
    out = {
        "f32": torch.zeros(300, 77, dtype=torch.bfloat16, device="cuda"),
        "bf16": torch.zeros(4099, dtype=torch.float32, device="cuda"),
        "f16": torch.zeros(48, 64, dtype=torch.bfloat16, device="cuda").t(),
        "f64": torch.zeros(30, 7, dtype=torch.float64, device="cuda"),  # fp32 -> fp64: stock path
        "ids": torch.zeros(33, 7, dtype=torch.int32, device="cuda"),  # integer conversion: stock path
        "same": torch.zeros(129, 3, device="cuda"),
        "meta": {"lr": 0.0},
    }
    dcp.load(out, storage_reader=CachedMetadataFileSystemReader(str(tmp_path / "ck"), load_on_engine=True))
    assert out["meta"] == sd["meta"]
    for k, v in out.items():
        if k != "meta":
            assert tensors_nan_aware_equal(v.cpu(), sd[k].cpu().to(v.dtype)), k


@pytest.mark.parametrize("pair", PAIRS, ids=_PAIR_IDS)
def test_budget_forced_split_with_conversion(tmp_path, built_library, monkeypatch, pair):
    from nvidia_resiliency_ext.checkpointing.b200.engine import SnapshotEngine

    src, dst = pair
    sd = _state(src)
    dcp.save(sd, checkpoint_id=str(tmp_path / "ck"))
    ref = _stock(tmp_path / "ck", sd, dst)
    monkeypatch.setattr(SnapshotEngine, "DCP_LOAD_STAGING", 256 << 10)  # "w" alone is 1.5-3 MB
    got = _engine(tmp_path / "ck", sd, dst, contiguous=False)
    stats = SnapshotEngine.get().last_box_load
    assert stats["batches"] > 5 and stats["peak_staging_bytes"] <= 256 << 10
    _assert_same(got, ref)


def test_checkpoint_written_by_the_async_writer(tmp_path, built_library, dist_1rank):
    from nvidia_resiliency_ext.checkpointing.async_ckpt.core import AsyncCallsQueue, AsyncRequest
    from nvidia_resiliency_ext.checkpointing.async_ckpt.filesystem_async import FileSystemWriterAsync
    from nvidia_resiliency_ext.checkpointing.async_ckpt.state_dict_saver import (
        save_state_dict_async_finalize,
        save_state_dict_async_plan,
    )

    sd = {}
    for dt in (torch.float32, torch.bfloat16, torch.float16):
        sd.update({f"{str(dt)[6:]}.{k}": v for k, v in _state(dt).items() if k != "t"})  # the writer takes contiguous tensors
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
    # every item into the next dtype of the cycle fp32 -> bf16 -> fp16 -> fp32
    nxt = {torch.float32: torch.bfloat16, torch.bfloat16: torch.float16, torch.float16: torch.float32}
    from nvidia_resiliency_ext.checkpointing.async_ckpt.cached_metadata_filesystem_reader import CachedMetadataFileSystemReader

    ref = {k: torch.zeros(v.shape, dtype=nxt[v.dtype]) for k, v in sd.items()}
    dcp.load(ref, storage_reader=FileSystemReader(str(tmp_path / "ck")))
    got = {k: torch.zeros(v.shape, dtype=nxt[v.dtype], device="cuda") for k, v in sd.items()}
    CachedMetadataFileSystemReader.clear_metadata_cache()
    dcp.load(got, storage_reader=CachedMetadataFileSystemReader(str(tmp_path / "ck"), load_on_engine=True))
    torch.cuda.synchronize()
    _assert_same(got, ref)
