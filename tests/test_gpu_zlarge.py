"""Tensors, records, boxes and checksum extents past 4 GiB, checked byte by byte on one GPU.

Every byte offset of the hot path is 64-bit: tile offsets of the pack / scatter walkers, box tiles and row addresses, CRC
extents, the pipelined snapshot's chunks and progress word, file extents of a restore, and the zip64 records of a
checkpoint container.  The other GPU tests stay below 2^32 bytes everywhere, where a 32-bit wrap of any of them is
invisible; a wrap inside one allocation gives wrong bytes rather than a fault.  Every test here asserts, before it
launches, that its geometry reaches past 2^32 bytes (from the planner's own tile lists, the extents or the file layout).

Inputs are seeded and generated on the device in pieces of at most 256 MiB, so the reference is regenerated piece by piece
and never held whole or copied to the host (the CRC data excepted: zlib needs it on the host).  Every byte is compared at
its own position, on the device, with ``torch.equal``; a mismatch reports how many bytes are wrong and the first wrong
offset.  Staging gaps, a guard behind every used range and destination bytes outside a box hold a sentinel that is checked
as well.

The ``zl`` fixture skips a test when the machine lacks the HBM, host memory or /dev/shm it needs (with the numbers in the
message), frees everything at teardown and prints each test's wall time and peak use."""
import ctypes as C
import gc
import io
import os
import shutil
import struct
import time
import zipfile
import zlib

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

TWO32 = 1 << 32
MIB, GIB = 1 << 20, 1 << 30
PIECE = 256 * MIB  # generation and comparison granule
SENTINEL = 0xA5
HOST_SENTINEL = 0x3C
GUARD = 512
LDG, TMA = 1, 2
VARIANTS = {"ldg": LDG, "tma": TMA}


# ---------------------------------------------------------------------------------------------------------------------
# resources
# ---------------------------------------------------------------------------------------------------------------------
def _meminfo(key):
    with open("/proc/meminfo") as f:
        for line in f:
            if line.startswith(key + ":"):
                return int(line.split()[1]) * 1024
    return 0


def _shm_free():
    try:
        st = os.statvfs("/dev/shm")
    except OSError:
        return 0
    return st.f_bavail * st.f_frsize


def _shm_used():
    try:
        st = os.statvfs("/dev/shm")
    except OSError:
        return 0
    return (st.f_blocks - st.f_bfree) * st.f_frsize


class _Resources:
    MARGIN = {"hbm": 2 * GIB, "ram": 2 * GIB, "shm": GIB}

    def __init__(self, name):
        self.name = name
        self.t0 = None
        self.shm0 = _shm_used()
        self.shm_peak = 0

    def need(self, hbm=0, ram=0, shm=0):
        """Skip unless the machine has these many bytes of free HBM, MemAvailable and free /dev/shm, plus a margin."""
        gc.collect()
        torch.cuda.empty_cache()
        have = {"hbm": torch.cuda.mem_get_info()[0], "ram": _meminfo("MemAvailable"), "shm": _shm_free()}
        want = {"hbm": hbm, "ram": ram, "shm": shm}
        short = [f"{k}: needs {(want[k] + self.MARGIN[k]) / GIB:.1f} GiB, has {have[k] / GIB:.1f} GiB"
                 for k in want if want[k] and have[k] < want[k] + self.MARGIN[k]]
        if short:
            pytest.skip("not enough memory for a >4 GiB test (" + "; ".join(short) + ")")
        torch.cuda.reset_peak_memory_stats()
        self.shm0 = _shm_used()
        self.t0 = time.perf_counter()

    def sample(self):
        self.shm_peak = max(self.shm_peak, _shm_used() - self.shm0)

    def finish(self):
        gc.collect()
        if torch.cuda.is_available():
            torch.cuda.synchronize()
            torch.cuda.empty_cache()
        if self.t0 is not None:
            print(f"\n[zlarge] {self.name}: {time.perf_counter() - self.t0:.1f} s, peak HBM allocated "
                  f"{torch.cuda.max_memory_allocated() / GIB:.2f} GiB, peak /dev/shm {self.shm_peak / GIB:.2f} GiB")


@pytest.fixture
def zl(request, built_library):
    res = _Resources(request.node.name)
    yield res
    res.finish()


# ---------------------------------------------------------------------------------------------------------------------
# seeded patterns, generated and compared piece by piece on the device
# ---------------------------------------------------------------------------------------------------------------------
def _gen(seed, k):
    return torch.Generator(device="cuda").manual_seed(seed * 1_000_003 + k)


def _byte_piece(seed, k, n):
    """Bytes [k * PIECE, k * PIECE + n) of byte pattern ``seed``."""
    return torch.randint(0, 256, (n,), dtype=torch.uint8, device="cuda", generator=_gen(seed, k))


def _f32_piece(seed, k, n):
    """Elements [k * PIECE / 4, + n) of fp32 pattern ``seed``: finite normal values."""
    return torch.randn(n, device="cuda", generator=_gen(seed, k))


def _pieces(n, per=PIECE):
    for k, lo in enumerate(range(0, n, per)):
        yield k, lo, min(per, n - lo)


def _u8(t):
    return t.reshape(-1).view(torch.uint8)


def _fill_bytes(flat_u8, seed):
    for k, lo, m in _pieces(flat_u8.numel()):
        flat_u8[lo:lo + m].copy_(_byte_piece(seed, k, m))


def _fill_f32(flat, seed):
    for k, lo, m in _pieces(flat.numel(), PIECE // 4):
        flat[lo:lo + m].copy_(_f32_piece(seed, k, m))


def _expect_equal(got, want, what, base=0):
    """Bytes of ``got`` equal ``want`` (a tensor of the same bytes, or one byte value), compared on the device."""
    got = _u8(got)
    if isinstance(want, int):
        ok = bool((got == want).all())
        ne = None if ok else got != want
    else:
        want = _u8(want.to(got.device) if want.device != got.device else want)
        assert got.numel() == want.numel(), f"{what}: {got.numel()} bytes, want {want.numel()}"
        ok = torch.equal(got, want)
        ne = None if ok else got != want
    if not ok:
        bad = int(ne.sum())
        first = int(torch.argmax(ne.to(torch.uint8)))
        raise AssertionError(f"{what}: {bad} wrong bytes in [{base}, {base + got.numel()}), first at byte {base + first}")


def _expect_fill(t_u8, value, what, base=0):
    for _, lo, m in _pieces(t_u8.numel()):
        _expect_equal(t_u8[lo:lo + m], value, what, base + lo)


def _expect_bytes(got_u8, seed, what, base=0):
    """``got_u8`` (uint8, on the device or the host) holds byte pattern ``seed`` from its first byte."""
    for k, lo, m in _pieces(got_u8.numel()):
        _expect_equal(got_u8[lo:lo + m].to("cuda"), _byte_piece(seed, k, m), what, base + lo)


def _expect_f32(got_flat, seed, what, conv=None):
    """``got_flat`` holds fp32 pattern ``seed`` (converted by ``conv``, a function of a device piece) element by element."""
    conv = conv or (lambda x: x)
    es = got_flat.element_size()
    for k, lo, m in _pieces(got_flat.numel(), PIECE // 4):
        _expect_equal(got_flat[lo:lo + m].to("cuda"), conv(_f32_piece(seed, k, m)), what, lo * es)


def _dev():
    return torch.cuda.current_device()


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _filled(nbytes, value=SENTINEL):
    return torch.full((nbytes,), value, dtype=torch.uint8, device="cuda")


def _round(v, a):
    return -(-v // a) * a


def _plan(tensors, flags=None, **kw):
    from nvidia_resiliency_ext.checkpointing.b200.engine import Plan

    ptrs = [t.data_ptr() if t.numel() else 0 for t in tensors]
    nbytes = [t.numel() * t.element_size() for t in tensors]
    return Plan(ptrs, nbytes, flags, device=_dev(), **kw)


def _expect_staging(stg, plan, segments, what):
    """Every segment of ``stg`` as ``segments[i](u8 slice, base)`` checks it, every gap and the guard still the sentinel."""
    cur = 0
    for i, (off, nb) in enumerate(zip(plan.offsets, plan.packed_nbytes)):
        if not nb:
            continue
        _expect_fill(stg[cur:off], SENTINEL, f"{what}: gap before segment {i}", cur)
        segments[i](stg[off:off + nb], off)
        cur = off + nb
    _expect_fill(stg[cur:], SENTINEL, f"{what}: gap / guard behind the last segment", cur)


# ---------------------------------------------------------------------------------------------------------------------
# A. pack and scatter through Plan, both walkers
# ---------------------------------------------------------------------------------------------------------------------
BIG = TWO32 + 3 * MIB + 4133  # bulk tiles and a 5-byte ragged tail past 2^32 when 16-byte aligned


def _bitcopy_state(mis):
    """(tensors, seeds): one BIG segment at ``mis`` bytes past a 16-byte boundary, then a 4-byte step, 13 bytes at an odd
    address and 1 MiB of fp32, whose staging offsets are past 2^32."""
    big = torch.empty(BIG + 16, dtype=torch.uint8, device="cuda")[mis:mis + BIG]
    step = torch.empty(1, device="cuda")
    odd = torch.empty(32, dtype=torch.uint8, device="cuda")[1:14]
    mb = torch.empty(MIB // 4, device="cuda")
    tensors, seeds = [big, step, odd, mb], [11, 12, 13, 14]
    for t, s in zip(tensors, seeds):
        _fill_bytes(_u8(t), s)
    assert big.data_ptr() % 16 == mis and odd.data_ptr() % 2 == 1
    return tensors, seeds


BITCOPY_CASES = [("ldg", 0, 0), ("tma", 0, 0), ("ldg", 3, 0), ("tma", 3, 0), ("tma", 0, 4096)]


@pytest.mark.parametrize("variant,mis,tile", BITCOPY_CASES, ids=[f"{v}-mis{m}-tile{t or 'default'}" for v, m, t in BITCOPY_CASES])
def test_pack_and_scatter_past_4gib(zl, variant, mis, tile):
    zl.need(hbm=2 * BIG + GIB)
    tensors, seeds = _bitcopy_state(mis)
    plan = _plan(tensors, tile_bytes=tile, variant=VARIANTS[variant])
    n_bulk, tiles = plan.tiles()
    past = [(i, t) for i, t in enumerate(tiles) if t[0] == 0 and t[2] >= TWO32]
    assert past, "segment 0 must have tiles whose offset is past 2^32"
    if mis == 0:
        assert any(i < n_bulk for i, _ in past) and any(i >= n_bulk for i, _ in past), "bulk tiles and a ragged tail past 2^32"
    assert all(o > TWO32 for o in plan.offsets[1:]), plan.offsets
    if tile == 4096:
        assert len(tiles) > 1 << 20
    total = plan.staging_bytes
    stg = _filled(total + GUARD)
    plan.pack(stg.data_ptr(), _stream())
    torch.cuda.synchronize()
    checks = [lambda s, b, seed=seed, i=i: _expect_bytes(s, seed, f"pack segment {i}", b) for i, seed in enumerate(seeds)]
    _expect_staging(stg, plan, checks, f"{variant} pack")

    # scatter into the zeroed sources: same pointers, same tile list
    for t in tensors:
        t.zero_()
    plan.scatter(stg.data_ptr(), _stream())
    torch.cuda.synchronize()
    for i, (t, seed) in enumerate(zip(tensors, seeds)):
        _expect_bytes(_u8(t), seed, f"{variant} scatter segment {i}")
    _expect_staging(stg, plan, checks, f"{variant} staging after the scatter")
    plan.close()


NARROW_LEAD = TWO32 // 2 + 4 * MIB + 48  # bit copy in front: the narrowed segment's packed range crosses 2^32
NARROW_ELEMS = (TWO32 + 64 * 1024 + 4) // 4  # fp32 elements: tensor-side offsets past 2^32


def _bf16_bits(x):
    return x.to(torch.bfloat16)


@pytest.mark.parametrize("variant", ["ldg", "tma"])
def test_narrow_pack_and_widen_scatter_past_4gib(zl, variant):
    zl.need(hbm=NARROW_LEAD + 4 * NARROW_ELEMS + 2 * NARROW_ELEMS + NARROW_LEAD + GIB)
    lead = torch.empty(NARROW_LEAD, dtype=torch.uint8, device="cuda")
    f32 = torch.empty(NARROW_ELEMS, device="cuda")
    _fill_bytes(lead, 21)
    _fill_f32(f32, 22)
    plan = _plan([lead, f32], flags=[0, 1], variant=VARIANTS[variant])
    off, packed = plan.offsets[1], plan.packed_nbytes[1]
    assert packed == 2 * NARROW_ELEMS and off < TWO32 < off + packed, "the packed bf16 range must cross 2^32 in staging"
    assert max(t[2] for t in plan.tiles()[1] if t[0] == 1) >= TWO32, "tensor-side offsets must pass 2^32"
    stg = _filled(plan.staging_bytes + GUARD)
    plan.pack(stg.data_ptr(), _stream())
    torch.cuda.synchronize()
    # the project's narrowing is torch's fp32 -> bf16 conversion on the device (RNE)
    checks = [lambda s, b: _expect_bytes(s, 21, "lead segment", b),
              lambda s, b: _expect_f32(s.view(torch.bfloat16), 22, "narrowed segment", _bf16_bits)]
    _expect_staging(stg, plan, checks, f"{variant} narrow pack")

    lead.zero_()
    f32.zero_()
    plan.scatter(stg.data_ptr(), _stream())
    torch.cuda.synchronize()
    _expect_bytes(lead, 21, "lead after the scatter")
    _expect_f32(f32, 22, "widened segment", lambda x: x.to(torch.bfloat16).to(torch.float32))  # widening is exact
    _expect_staging(stg, plan, checks, f"{variant} staging after the widen scatter")
    plan.close()


# ---------------------------------------------------------------------------------------------------------------------
# B. pipelined snapshot into a pinned host buffer larger than 4 GiB
# ---------------------------------------------------------------------------------------------------------------------
def _expected_launches(total, chunk, growth):
    """nvrx_snapshot's group rule: chunks of round_up(chunk, 512) bytes (at most 256); pack launches cover 1, g, g^2, ..."""
    if chunk == 0 or chunk > total:
        chunk = total if total else 1
    chunk = _round(chunk, 512)
    n = -(-total // chunk) if total else 0
    if n > 256:
        chunk = _round(-(-total // 256), 512)
        n = -(-total // chunk)
    launches, c, group = 0, 0, 1
    while c < n:
        c = min(n, c + group)
        launches += 1
        group *= growth
    return launches


@pytest.mark.parametrize("variant", ["ldg", "tma"])
def test_pipelined_snapshot_into_a_host_buffer_past_4gib(zl, monkeypatch, variant):
    from nvidia_resiliency_ext.checkpointing.b200 import _cabi
    from nvidia_resiliency_ext.checkpointing.b200.engine import HostBuffer

    zl.need(hbm=2 * BIG + GIB, ram=BIG + GIB)
    monkeypatch.delenv("NVRX_B200_PACK_GROWTH", raising=False)  # the default growth, 4
    tensors, seeds = _bitcopy_state(0)
    plan = _plan(tensors, variant=VARIANTS[variant])
    total = plan.staging_bytes
    chunk = 256 * MIB
    stg = _filled(total + GUARD)
    hb = HostBuffer.create(total + GUARD, pin=True, device=_dev())
    host = hb.as_tensor(total + GUARD)
    assert hb.capacity > TWO32
    drain = torch.cuda.Stream()
    base = 3 << 33  # a progress word truncated to 32 bits anywhere differs
    try:
        host.fill_(HOST_SENTINEL)
        torch.cuda.synchronize()
        _cabi.check(_cabi.lib().nvrx_snapshot(plan._h, stg.data_ptr(), hb.data_ptr, chunk, hb.progress_ptr, base, _stream(),
                                              drain.cuda_stream, None, None), "nvrx_snapshot")
        torch.cuda.synchronize()
        assert hb.progress == base + total and hb.progress >= TWO32
        assert plan.last_launches() == _expected_launches(total, chunk, 4) == 3
        checks = [lambda s, b, t=t: _expect_equal(s, _u8(t), "staging", b) for t in tensors]
        _expect_staging(stg, plan, checks, "snapshot staging")
        # the host copy: segments against the device sources, gaps as staging had them, nothing written past the end
        cur = 0
        for i, (t, off, nb) in enumerate(zip(tensors, plan.offsets, plan.packed_nbytes)):
            for _, lo, m in _pieces(off - cur):
                _expect_equal(host[cur + lo:cur + lo + m].cuda(), SENTINEL, f"host gap before segment {i}", cur + lo)
            src = _u8(t)
            for _, lo, m in _pieces(nb):
                _expect_equal(host[off + lo:off + lo + m].cuda(), src[lo:lo + m], f"host segment {i}", off + lo)
            cur = off + nb
        _expect_equal(host[cur:total].cuda(), SENTINEL, "host padding", cur)
        _expect_equal(host[total:].cuda(), HOST_SENTINEL, "host guard", total)
    finally:
        plan.close()
        del host
        hb.close()


# ---------------------------------------------------------------------------------------------------------------------
# C. checksums
# ---------------------------------------------------------------------------------------------------------------------
CRC_LEN = TWO32 + GIB + 4096
CRC_SENTINEL = 0x5A5A5A5A


def _host_random(n, seed):
    rng = np.random.default_rng(seed)
    words = rng.integers(0, 1 << 63, size=-(-n // 8), dtype=np.uint64)
    return words.view(np.uint8)[:n]


def test_crc_extents_past_4gib(zl):
    from nvidia_resiliency_ext.checkpointing.b200.engine import CrcPlan, CrcxPlan, finish_crcs

    zl.need(hbm=CRC_LEN + GIB, ram=CRC_LEN + 2 * GIB)
    host = _host_random(CRC_LEN, 31)
    dev = torch.empty(CRC_LEN, dtype=torch.uint8, device="cuda")
    for _, lo, m in _pieces(CRC_LEN):
        dev[lo:lo + m].copy_(torch.from_numpy(host[lo:lo + m]))
    torch.cuda.synchronize()
    # any offset and length (CrcxPlan): a long one from byte 5, one past 2^32, one across it, an empty one past it
    offsets = [5, TWO32 + 3, TWO32 - 9, TWO32 + 100]
    nbytes = [TWO32 + 777, GIB + 13, 3 * MIB + 1001, 0]
    assert offsets[0] + nbytes[0] > TWO32 and nbytes[0] >= TWO32 and offsets[1] >= TWO32
    assert offsets[2] < TWO32 < offsets[2] + nbytes[2]
    assert all(o + n <= CRC_LEN for o, n in zip(offsets, nbytes))
    want = [zlib.crc32(memoryview(host)[o:o + n]) for o, n in zip(offsets, nbytes)]
    plan = CrcxPlan(offsets, nbytes, _dev())
    vals = torch.full((len(offsets) + 8,), CRC_SENTINEL, dtype=torch.int32).pin_memory()
    plan.run(dev.data_ptr(), vals.data_ptr(), _stream())
    torch.cuda.synchronize()
    got = [v & 0xFFFFFFFF for v in vals.tolist()]
    plan.close()
    assert got[:len(offsets)] == want, [(o, n) for o, n, g, w in zip(offsets, nbytes, got, want) if g != w]
    assert got[len(offsets):] == [CRC_SENTINEL] * 8

    # the record checksum of the snapshot path (CrcPlan + finish_crcs): aligned extents, one longer than 2^32, one past it
    offsets, nbytes = [16, TWO32 + 512], [TWO32 + 777, GIB - 512 + 13]
    assert nbytes[0] > TWO32 and offsets[1] > TWO32 and all(o + n <= CRC_LEN for o, n in zip(offsets, nbytes))
    want = [zlib.crc32(memoryview(host)[o:o + n]) for o, n in zip(offsets, nbytes)]
    plan = CrcPlan(offsets, nbytes, _dev())
    values = torch.zeros(plan.n_values + 2, dtype=torch.int32).pin_memory()
    ready = torch.zeros(1, dtype=torch.int64).pin_memory()
    plan.run(dev.data_ptr(), values.data_ptr(), ready.data_ptr(), 7, _stream())
    torch.cuda.synchronize()
    assert int(ready[0]) == 7
    assert finish_crcs(offsets, nbytes, values.data_ptr(), plan.n_values, host.ctypes.data) == want
    plan.close()


# ---------------------------------------------------------------------------------------------------------------------
# D. box scatter through BoxPlan
# ---------------------------------------------------------------------------------------------------------------------
def _boxplan(boxes, staging_bytes, casts=None):
    from nvidia_resiliency_ext.checkpointing.b200.engine import BoxPlan

    return BoxPlan(boxes, staging_bytes, device=_dev(), casts=casts)


def _rows_reaching(tiles, row_bytes_dst):
    """Largest byte distance from the box's base that a multi-row tile's rows reach, on the side with ``row_bytes_dst``."""
    return max((t[1] + t[2] - 1) * row_bytes_dst for t in tiles if t[2] > 1)


RUN_BYTES = TWO32 + 5 * MIB + 77
COL_ROWS = TWO32 // (1100 * 4) + 64  # rows x 1100 fp32 > 4 GiB
SHORT_STRIDE = 4099  # fp32 elements between the 3-element rows of the short-row box
SHORT_ROWS = TWO32 // (SHORT_STRIDE * 4) + 33


@pytest.mark.parametrize("shape", ["run", "columns", "short_rows"])
def test_box_copy_past_4gib(zl, shape):
    """One box per tile shape, each reaching more than 2^32 bytes past its base: a single run cut into byte ranges, a
    column box of 2000-byte rows (a warp per row) and 12-byte rows (a thread per row)."""
    if shape == "run":
        zl.need(hbm=2 * RUN_BYTES + GIB)
        so, do = 5, 11
        stg = torch.empty(so + RUN_BYTES, dtype=torch.uint8, device="cuda")
        _fill_bytes(stg, 41)
        dst = _filled(do + RUN_BYTES + GUARD)
        box = (1, [RUN_BYTES], so, [1], dst.data_ptr() + do, [1])
        bp = _boxplan([box], stg.numel())
        tiles = bp.tiles()
        assert all(t[2] == 1 for t in tiles) and max(t[3] for t in tiles) >= TWO32, "byte ranges of one row past 2^32"
        bp.scatter(stg.data_ptr(), _stream())
        torch.cuda.synchronize()
        _expect_fill(dst[:do], SENTINEL, "before the box")
        for _, lo, m in _pieces(RUN_BYTES):
            _expect_equal(dst[do + lo:do + lo + m], stg[so + lo:so + lo + m], "run", do + lo)
        _expect_fill(dst[do + RUN_BYTES:], SENTINEL, "guard", do + RUN_BYTES)
    else:
        if shape == "columns":
            rows, cols, width, c0 = COL_ROWS, 1100, 500, 300
        else:
            rows, cols, width, c0 = SHORT_ROWS, SHORT_STRIDE, 3, 0
        zl.need(hbm=rows * cols * 4 + rows * width * 4 + GIB)
        stg = torch.empty(rows * width * 4, dtype=torch.uint8, device="cuda")
        _fill_bytes(stg, 42)
        dst = _filled(rows * cols * 4 + GUARD)
        box = (4, [rows, width], 0, [width, 1], dst.data_ptr() + c0 * 4, [cols, 1])
        bp = _boxplan([box], stg.numel())
        tiles = bp.tiles()
        assert width * 4 >= 32 if shape == "columns" else width * 4 < 32
        assert any(t[2] > 1 for t in tiles) and _rows_reaching(tiles, cols * 4) >= TWO32, "rows past 2^32 of the destination"
        bp.scatter(stg.data_ptr(), _stream())
        torch.cuda.synchronize()
        d2 = dst[:rows * cols * 4].view(rows, cols * 4)
        s2 = stg.view(rows, width * 4)
        step = max(1, PIECE // (cols * 4))
        for r0 in range(0, rows, step):
            r1 = min(rows, r0 + step)
            blk = d2[r0:r1]
            _expect_equal(blk[:, c0 * 4:(c0 + width) * 4].contiguous(), s2[r0:r1], f"box rows {r0}..{r1}", r0 * cols * 4)
            _expect_fill(blk[:, :c0 * 4].contiguous().view(-1), SENTINEL, f"left of the box, rows {r0}..{r1}")
            _expect_fill(blk[:, (c0 + width) * 4:].contiguous().view(-1), SENTINEL, f"right of the box, rows {r0}..{r1}")
        _expect_fill(dst[rows * cols * 4:], SENTINEL, "guard")
    _expect_bytes(stg, 41 if shape == "run" else 42, "staging after the scatter")
    bp.close()


CAST_RUN_BF16 = (TWO32 + 4 * MIB) // 4 + 5  # bf16 elements: source bytes < 2^32, destination fp32 bytes > 2^32
CAST_RUN_F32 = (TWO32 + 4 * MIB) // 4 + 3  # fp32 elements: source bytes > 2^32


def _tie_to_oracle(code, src_first, ref_first):
    """torch's conversion equals the project's oracle on the first MiB of the pattern."""
    from _cast_oracle import convert_bits

    u = {2: np.uint16, 4: np.uint32}
    s = src_first.cpu().contiguous().view(torch.int16 if src_first.element_size() == 2 else torch.int32).numpy().view(u[src_first.element_size()])
    r = ref_first.cpu().contiguous().view(torch.int16 if ref_first.element_size() == 2 else torch.int32).numpy().view(u[ref_first.element_size()])
    assert np.array_equal(convert_bits(code, s.reshape(-1)).astype(r.dtype), r.reshape(-1))


@pytest.mark.parametrize("case", ["bf16_to_f32_run", "f32_to_bf16_run", "f32_to_bf16_rows"])
def test_box_cast_past_4gib(zl, case):
    from nvidia_resiliency_ext.checkpointing.b200 import _cabi

    if case == "bf16_to_f32_run":
        n = CAST_RUN_BF16
        zl.need(hbm=6 * n + GIB)
        stg = torch.empty(n, dtype=torch.bfloat16, device="cuda")
        for k, lo, m in _pieces(n, PIECE // 4):
            stg[lo:lo + m].copy_(_f32_piece(51, k, m).to(torch.bfloat16))
        dst = _filled(4 * n + GUARD)
        code = _cabi.CAST_BF16_F32
        bp = _boxplan([(2, [n], 0, [1], dst.data_ptr(), [1])], 2 * n, casts=[code])
        tiles = bp.tiles()
        assert all(t[2] == 1 for t in tiles)
        assert max(t[3] + t[4] for t in tiles) <= TWO32 < max(t[3] // 2 * 4 for t in tiles), "source below, destination past 2^32"
        _tie_to_oracle(code, stg[:MIB // 2], stg[:MIB // 2].to(torch.float32))
        bp.scatter(stg.data_ptr(), _stream())
        torch.cuda.synchronize()
        out = dst[:4 * n].view(torch.float32)
        for k, lo, m in _pieces(n, PIECE // 4):
            _expect_equal(out[lo:lo + m], _f32_piece(51, k, m).to(torch.bfloat16).to(torch.float32), "bf16 -> fp32 run", 4 * lo)
        _expect_fill(dst[4 * n:], SENTINEL, "guard", 4 * n)
    elif case == "f32_to_bf16_run":
        n = CAST_RUN_F32
        zl.need(hbm=6 * n + GIB)
        stg = torch.empty(n, device="cuda")
        _fill_f32(stg, 52)
        dst = _filled(2 * n + GUARD)
        code = _cabi.CAST_F32_BF16
        bp = _boxplan([(4, [n], 0, [1], dst.data_ptr(), [1])], 4 * n, casts=[code])
        tiles = bp.tiles()
        assert all(t[2] == 1 for t in tiles) and max(t[3] for t in tiles) >= TWO32, "source byte ranges past 2^32"
        _tie_to_oracle(code, stg[:MIB // 4], stg[:MIB // 4].to(torch.bfloat16))
        bp.scatter(stg.data_ptr(), _stream())
        torch.cuda.synchronize()
        _expect_f32(dst[:2 * n].view(torch.bfloat16), 52, "fp32 -> bf16 run", _bf16_bits)
        _expect_fill(dst[2 * n:], SENTINEL, "guard", 2 * n)
    else:
        rows, cols, width, c0 = COL_ROWS, 1100, 500, 300
        zl.need(hbm=rows * cols * 4 + rows * width * 2 + GIB)
        stg = torch.empty(rows * cols, device="cuda")
        _fill_f32(stg, 53)
        dst = _filled(rows * width * 2 + GUARD)
        code = _cabi.CAST_F32_BF16
        bp = _boxplan([(4, [rows, width], c0 * 4, [cols, 1], dst.data_ptr(), [width, 1])], stg.numel() * 4, casts=[code])
        tiles = bp.tiles()
        assert any(t[2] > 1 for t in tiles) and _rows_reaching(tiles, cols * 4) >= TWO32, "source rows past 2^32 (a warp per row)"
        s2 = stg.view(rows, cols)
        _tie_to_oracle(code, s2[:512, c0:c0 + width], s2[:512, c0:c0 + width].to(torch.bfloat16))
        bp.scatter(stg.data_ptr(), _stream())
        torch.cuda.synchronize()
        d2 = dst[:rows * width * 2].view(torch.bfloat16).view(rows, width)
        step = PIECE // (cols * 4)
        for r0 in range(0, rows, step):
            r1 = min(rows, r0 + step)
            _expect_equal(d2[r0:r1], s2[r0:r1, c0:c0 + width].to(torch.bfloat16), f"cast rows {r0}..{r1}", r0 * width * 2)
        _expect_fill(dst[rows * width * 2:], SENTINEL, "guard", rows * width * 2)
    bp.close()


# ---------------------------------------------------------------------------------------------------------------------
# E. the engine end to end with one tensor over 4 GiB
# ---------------------------------------------------------------------------------------------------------------------
EMB_SHAPE = (262147, 4096)  # fp32: 4,295,016,448 bytes
EMB_BYTES = EMB_SHAPE[0] * EMB_SHAPE[1] * 4


def _engine_state():
    emb = torch.empty(EMB_SHAPE, device="cuda")
    _fill_f32(emb.view(-1), 61)
    g = torch.Generator(device="cuda").manual_seed(62)
    return {"emb": emb, "step": torch.tensor(12345.0, device="cuda"),
            "ids": torch.randint(-(1 << 40), 1 << 40, (1001,), device="cuda", generator=g),
            "half": torch.randn(3333, device="cuda", generator=g).to(torch.bfloat16)}


def _expect_state(got, want, what):
    assert list(got) == list(want), what
    for k in want:
        assert got[k].dtype == want[k].dtype and got[k].shape == want[k].shape, (what, k)
        if k == "emb":
            _expect_f32(got[k].reshape(-1), 61, f"{what}: emb")
        else:
            _expect_equal(got[k].to("cuda"), want[k], f"{what}: {k}")


def _zip64_extra(extra):
    """The zip64 extended-information field (id 0x0001) of an extra block, or None."""
    i = 0
    while i + 4 <= len(extra):
        hid, size = struct.unpack_from("<HH", extra, i)
        if hid == 1:
            return extra[i + 4:i + 4 + size]
        i += 4 + size
    return None


def _expect_zip64_container(path, local_zip64):
    """The record over 4 GiB is data/0 with zip64 fields in its central directory entry (and, ``local_zip64``, in its
    local header); every other record sits past 4 GiB; every record passes its CRC check (streamed)."""
    with zipfile.ZipFile(path) as zf:
        infos = zf.infolist()
        big = [zi for zi in infos if zi.file_size >= TWO32]
        assert len(big) == 1 and big[0].filename.endswith("/data/0"), [zi.filename for zi in big]
        zi = big[0]
        assert _zip64_extra(zi.extra) is not None, "central directory entry of data/0 is not zip64"
        if local_zip64:
            with open(path, "rb") as f:
                f.seek(zi.header_offset)
                hdr = f.read(30)
                sig, csize, usize = struct.unpack_from("<I14xII", hdr)
                nlen, xlen = struct.unpack_from("<HH", hdr, 26)
                f.seek(zi.header_offset + 30 + nlen)
                extra = f.read(xlen)
            assert sig == 0x04034B50 and csize == usize == 0xFFFFFFFF, "local header of data/0 must defer its sizes to zip64"
            z = _zip64_extra(extra)
            assert z is not None and struct.unpack_from("<QQ", z) == (zi.file_size, zi.file_size), "zip64 local sizes"
        records = [x for x in infos if "/data/" in x.filename and x is not zi and not x.filename.endswith("/.pad")]
        assert records and all(x.header_offset > TWO32 for x in records), "the small records must sit past 4 GiB"
        for x in infos:
            if x.filename.endswith("/.pad"):
                continue
            with zf.open(x) as r:  # raises BadZipFile on a wrong CRC-32 at the end of the record
                while r.read(64 * MIB):
                    pass
        return zi


@pytest.mark.parametrize("writer", ["zero_copy", "copying"])
def test_async_save_of_a_tensor_past_4gib(zl, shm_dir, dist_1rank, monkeypatch, writer):
    from nvidia_resiliency_ext.checkpointing.async_ckpt.torch_ckpt import TorchAsyncCheckpoint
    from nvidia_resiliency_ext.checkpointing.b200.engine import SnapshotEngine

    if not str(shm_dir).startswith("/dev/shm"):
        pytest.skip("needs /dev/shm")
    copies = 2 if writer == "copying" else 1
    zl.need(hbm=2 * EMB_BYTES + GIB, ram=EMB_BYTES + 2 * GIB, shm=copies * EMB_BYTES)
    monkeypatch.setenv("NVRX_B200_ZERO_COPY", "1" if writer == "zero_copy" else "0")
    monkeypatch.setenv("NVRX_B200_ZIP_CRC", "1")
    sd = _engine_state()
    path = shm_dir / "big.pt"
    ckpt = TorchAsyncCheckpoint(persistent_queue=False)
    try:
        ckpt.async_save(sd, path)
        ckpt.finalize_async_save(blocking=True)
        zl.sample()
        assert os.stat(path).st_nlink == (2 if writer == "zero_copy" else 1)
        assert os.path.getsize(path) > EMB_BYTES
        _expect_zip64_container(path, local_zip64=writer == "zero_copy")  # the slot container's own headers
        loaded = torch.load(path, weights_only=False, mmap=True)
        _expect_state(loaded, sd, f"{writer} torch.load(mmap=True)")
        del loaded
    finally:
        ckpt.close()
        if path.exists():
            path.unlink()
        SnapshotEngine.shutdown_all()


def test_local_manager_restore_past_4gib(zl, shm_dir, dist_1rank, monkeypatch):
    from nvidia_resiliency_ext.checkpointing.b200.engine import HostBuffer, SnapshotEngine
    from nvidia_resiliency_ext.checkpointing.local.basic_state_dict import BasicTensorAwareStateDict
    from nvidia_resiliency_ext.checkpointing.local.ckpt_managers.local_manager import LocalCheckpointManager

    zl.need(hbm=3 * EMB_BYTES + GIB, ram=EMB_BYTES + 2 * GIB, shm=EMB_BYTES)
    monkeypatch.setenv("NVRX_B200_ZERO_COPY", "1")
    monkeypatch.setenv("NVRX_B200_ZIP_CRC", "1")  # the record checksums NVRX_B200_VERIFY_RESTORE compares with
    sd = _engine_state()
    root = shm_dir / "local"
    try:
        LocalCheckpointManager(root).save(BasicTensorAwareStateDict(dict(sd)), 1, is_async=False)
        zl.sample()
        # a fresh process sees no resident slot.  Unverified, the restore reads the file straight into staging
        # (nvrx_fill_from_fd); verified, it reads the file into a pinned slot (readv) whose record checksums the GPU checks
        monkeypatch.setenv("NVRX_B200_ZERO_COPY", "0")
        eng = SnapshotEngine.get()
        real_fill, real_readv = eng.lib.nvrx_fill_from_fd, HostBuffer.readv_fd
        extents = []

        def spy_fill(stg, total, fd, n, stg_offs, nbytes, file_offs, *rest):
            extents.append(("fill_from_fd", total, [(stg_offs[i], nbytes[i], file_offs[i]) for i in range(n)]))
            return real_fill(stg, total, fd, n, stg_offs, nbytes, file_offs, *rest)

        def spy_readv(self, offsets, nbytes, file_offs, fd, **kw):
            extents.append(("readv", self.capacity, list(zip(offsets, nbytes, file_offs))))
            return real_readv(self, offsets, nbytes, file_offs, fd, **kw)

        monkeypatch.setattr(eng.lib, "nvrx_fill_from_fd", spy_fill)
        monkeypatch.setattr(HostBuffer, "readv_fd", spy_readv)
        for verify in ("0", "1"):
            monkeypatch.setenv("NVRX_B200_VERIFY_RESTORE", verify)
            mgr = LocalCheckpointManager(root)
            assert mgr.find_latest() == 1
            restores = eng.file_restores
            extents.clear()
            loaded, _ = mgr.load()
            assert eng.file_restores == restores + (verify == "0")
            (how, total, ext), = extents
            assert how == ("fill_from_fd" if verify == "0" else "readv"), how
            assert total > TWO32 and any(nb >= TWO32 for _, nb, _ in ext), "an extent of 4 GiB or more"
            assert any(fo > TWO32 for _, _, fo in ext) and any(so > TWO32 for so, _, _ in ext), "extents past 4 GiB"
            _expect_state(loaded.state_dict, sd, f"local restore verify={verify}")
            del loaded
            gc.collect()
    finally:
        SnapshotEngine.shutdown_all()


# ---------------------------------------------------------------------------------------------------------------------
# F. DCP load of a record over 4 GiB
# ---------------------------------------------------------------------------------------------------------------------
class _Window(io.RawIOBase):
    """Read-only file view of ``[base, base + length)``: zipfile on one archive embedded in a .distcp file."""

    def __init__(self, f, base, length):
        self.f, self.base, self.length, self.pos = f, base, length, 0

    def readable(self):
        return True

    def seekable(self):
        return True

    def seek(self, off, whence=0):
        self.pos = {0: off, 1: self.pos + off, 2: self.length + off}[whence]
        return self.pos

    def tell(self):
        return self.pos

    def read(self, n=-1):
        n = self.length - self.pos if n is None or n < 0 else min(n, self.length - self.pos)
        self.f.seek(self.base + self.pos)
        out = self.f.read(max(n, 0))
        self.pos += len(out)
        return out


def _dcp_targets(dtype):
    emb = torch.empty(EMB_SHAPE, dtype=dtype, device="cuda")
    _u8(emb).fill_(SENTINEL)
    return {"emb": emb, "tail": torch.zeros(777, dtype=torch.int64, device="cuda")}


def test_dcp_load_of_a_record_past_4gib(zl, shm_dir):
    import torch.distributed.checkpoint as dcp
    from torch.distributed.checkpoint import FileSystemReader
    from torch.distributed.checkpoint.api import CheckpointException

    from nvidia_resiliency_ext.checkpointing.async_ckpt.cached_metadata_filesystem_reader import CachedMetadataFileSystemReader
    from nvidia_resiliency_ext.checkpointing.b200.engine import SnapshotEngine
    from nvidia_resiliency_ext.checkpointing.b200.ptzip import read_tensor_record

    zl.need(hbm=EMB_BYTES + 3 * GIB, ram=EMB_BYTES + 2 * GIB, shm=EMB_BYTES)
    emb = torch.empty(EMB_SHAPE)
    flat = emb.view(-1)
    for k, lo, m in _pieces(flat.numel(), PIECE // 4):
        flat[lo:lo + m].copy_(_f32_piece(61, k, m).cpu())
    tail = torch.arange(777, dtype=torch.int64) * 1_000_003
    root = shm_dir / "dcp"
    dcp.save({"emb": emb, "tail": tail}, checkpoint_id=str(root))
    zl.sample()
    del emb, flat
    gc.collect()
    try:
        md = FileSystemReader(str(root)).read_metadata()
        item = next(v for k, v in md.storage_data.items() if k.fqn == "emb")
        path = os.path.join(str(root), item.relative_path)
        fd = os.open(path, os.O_RDONLY)
        try:
            rec = read_tensor_record(fd, item.offset, item.length)
        finally:
            os.close(fd)
        assert rec.record_len >= TWO32 and rec.record_len == EMB_BYTES
        with open(path, "rb") as f:
            with zipfile.ZipFile(_Window(f, item.offset, item.length)) as zf:
                zi = next(x for x in zf.infolist() if x.filename.endswith("/data/0"))
                assert zi.file_size == rec.record_len and _zip64_extra(zi.extra) is not None
                f.seek(item.offset + zi.header_offset)
                nlen, xlen = struct.unpack("<HH", f.read(30)[26:30])
            assert rec.data_off == item.offset + zi.header_offset + 30 + nlen + xlen
            assert rec.crc32 == zi.CRC != 0

        def load(dtype, verify):
            out = _dcp_targets(dtype)
            CachedMetadataFileSystemReader.clear_metadata_cache()
            dcp.load(out, storage_reader=CachedMetadataFileSystemReader(str(root), load_on_engine=True, verify=verify))
            torch.cuda.synchronize()
            return out, dict(SnapshotEngine.get().last_box_load)

        for verify in (False, True):
            out, stats = load(torch.float32, verify)
            assert stats["batches"] >= 3, stats  # the single run is cut into element ranges past 2^32 of the target
            if verify:
                assert stats["verified_records"] == 2 and stats["verify_extra_bytes"] == 0, stats
            _expect_f32(out["emb"].view(-1), 61, f"dcp load verify={verify}")
            _expect_equal(out["tail"], tail.cuda(), "tail")
            del out
        out, _ = load(torch.bfloat16, False)
        _expect_f32(out["emb"].view(-1), 61, "dcp load into bf16", _bf16_bits)
        del out

        at = rec.data_off + TWO32 + 4097
        assert at < rec.data_off + rec.record_len
        fd = os.open(path, os.O_RDWR)
        try:
            byte = os.pread(fd, 1, at)[0]
            os.pwrite(fd, bytes([byte ^ 0x01]), at)
            try:
                with pytest.raises(CheckpointException, match=r"(?s)crc32 mismatch.*emb"):
                    load(torch.float32, True)
            finally:
                os.pwrite(fd, bytes([byte]), at)
        finally:
            os.close(fd)
    finally:
        shutil.rmtree(root, ignore_errors=True)
        SnapshotEngine.shutdown_all()
