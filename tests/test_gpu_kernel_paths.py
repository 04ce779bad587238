"""Every launch path of the snapshot and box-scatter kernels, bit-exact on one GPU.

Each test fills staging, destinations and stand-in peer buffers with a sentinel byte, runs one path and compares every
byte of those buffers with a plain reference: the packed image of oracle/snapshot_oracle.py (or the same layout assembled
by byte slicing for the large states), or ``_box_oracle.box_copy`` for box scatter.  A wrong byte inside a segment, a write
into a segment gap or past a buffer's end, and a scatter that modifies its source all fail.

Which code runs is chosen through the settings the library reads at every launch (NVRX_B200_TMA_STAGES,
NVRX_B200_TMA_CTAS_PER_SM, NVRX_B200_LDG_CTAS_PER_SM, NVRX_B200_SHARD_INTERLEAVE, NVRX_B200_PACK_GROWTH).  Where a test
depends on a geometry (the TMA ring wrapping around, a shard edge inside a tensor, a chunk edge inside a tile) it asserts
that premise from the planner's own tile list before it launches anything."""
import ctypes as C

import numpy as np
import pytest
import torch

from _box_oracle import _contig_strides, _random_boxes, box_copy
from oracle import snapshot_oracle as orc

pytestmark = pytest.mark.gpu

LDG, TMA = 1, 2
VARIANTS = {"ldg": LDG, "tma": TMA}
SENTINEL = 0xA5  # staging, destinations, peer buffers
HOST_SENTINEL = 0x3C  # host buffer of the pipelined snapshot: a chunk copied before its pack shows up as 0xA5
GUARD = 512  # bytes behind every buffer's used range that must stay untouched


def _dev():
    return torch.cuda.current_device()


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _sm_count():
    from nvidia_resiliency_ext.checkpointing.b200 import _cabi

    n = C.c_int()
    _cabi.check(_cabi.lib().nvrx_device_info(_dev(), C.byref(n), None, None, 0), "nvrx_device_info")
    return n.value


def _round(v, a):
    return -(-v // a) * a


def _filled(nbytes, value=SENTINEL):
    return torch.full((nbytes,), value, dtype=torch.uint8, device="cuda")


def _ptrs(tensors):
    return [t.data_ptr() if t.numel() else 0 for t in tensors]


def _nbytes(tensors):
    return [t.numel() * t.element_size() for t in tensors]


def _plan(tensors, narrow=False, **kw):
    from nvidia_resiliency_ext.checkpointing.b200.engine import Plan

    flags = [1 if m else 0 for m in orc.narrow_mask(tensors, narrow)]
    return Plan(_ptrs(tensors), _nbytes(tensors), flags, device=_dev(), **kw)


def _image(pieces, length, sentinel=SENTINEL):
    """`length` sentinel bytes with each (offset, uint8 array) piece written over them."""
    img = np.full(length, sentinel, dtype=np.uint8)
    for off, raw in pieces:
        img[off : off + raw.size] = raw
    return img


def _packed_image(tensors, narrow=False, offsets=None, length=None):
    """Expected staging after a pack: the oracle's bytes at the segment ranges, sentinel in the gaps and behind the end.
    ``offsets``: caller-chosen segment offsets (a container layout) instead of the oracle's round-up rule."""
    if offsets is None:
        exp, offsets, packed = orc.pack_oracle(tensors, narrow)
        total = exp.size
        pieces = [(o, exp[o : o + n]) for o, n in zip(offsets, packed)]
    else:
        mask = orc.narrow_mask(tensors, narrow)
        pieces = []
        for t, o, nr in zip(tensors, offsets, mask):
            raw = orc.tensor_bytes(t)
            if nr:
                raw = orc.f32_bits_to_bf16_bits(raw.view(np.uint32)).view(np.uint8)
            pieces.append((o, raw))
        total = _round(max([o + r.size for o, r in pieces], default=0), orc.DEFAULT_ALIGN)
    return _image(pieces, total + GUARD if length is None else length), total


def _assert_bytes(got, want, what):
    got = got.cpu().numpy() if isinstance(got, torch.Tensor) else got
    assert got.shape == want.shape, what
    bad = np.flatnonzero(got != want)
    assert bad.size == 0, f"{what}: {bad.size} wrong bytes, first at {bad[0]} (got {got[bad[0]]:#x}, want {want[bad[0]]:#x})"


def _assert_equal_dev(got, want, what):
    """Device compare; the host copy is only made to describe a mismatch."""
    if not torch.equal(got, want):
        _assert_bytes(got.cpu().numpy(), want.cpu().numpy(), what)


def _carve(flat, segs):
    return [flat[o : o + n] for o, n in segs]


def _ring_layout(rng, tile, want_bulk):
    """(offset, nbytes) of segments carved from one flat buffer, and its used length.  Seven of every eight start 16-byte
    aligned and are 1 KiB .. 3 tiles long with a 0-15-byte tail, so bulk tiles of every length sit next to ragged tails; the
    eighth is misaligned and tiny (or, every 16th, up to 3 tiles of ragged work).  Segments are added until the planner's
    rule (aligned pieces of >= 1 KiB per tile are bulk tiles) gives ``want_bulk`` bulk tiles."""
    segs, cur, n_bulk = [], 0, 0
    while n_bulk < want_bulk:
        k = len(segs)
        if k % 8 == 7:
            cur = _round(cur, 16) + int(rng.integers(1, 16))
            nb = int(rng.integers(0, 3 * tile)) if k % 16 == 15 else int(rng.integers(0, 64))
        else:
            cur = _round(cur, 16)
            nb = int(rng.integers(1024 // 16, 3 * tile // 16 + 1)) * 16 + int(rng.integers(0, 16))
            n_bulk += sum(1 for o in range(0, nb, tile) if min(tile, nb - o) >= 1024)
        segs.append((cur, nb))
        cur += nb
    return segs, cur


def _same_class_destinations(segs, end):
    """Destination offsets of the same alignment class (mod 16) as the source offsets, each pushed 16 bytes further."""
    return [o + 16 * i for i, (o, _) in enumerate(segs)], end + 16 * len(segs)


# ---------------------------------------------------------------------------------------------------------------------
# a. the TMA ring wraps around: every launch_tma instantiation, pack and scatter, several times more tiles per CTA than stages
# ---------------------------------------------------------------------------------------------------------------------
def _ring_roundtrip(variant, tile, stages, grid, seed):
    rng = np.random.default_rng(seed)
    segs, end = _ring_layout(rng, tile, want_bulk=int(3.3 * stages * grid) + 1)
    g = torch.Generator(device="cuda").manual_seed(seed)
    flat = torch.randint(0, 256, (end + GUARD,), dtype=torch.uint8, device="cuda", generator=g)
    src = _carve(flat, segs)
    plan = _plan(src, tile_bytes=tile, variant=variant)
    n_bulk, tiles = plan.tiles()
    per_cta = (n_bulk if variant == TMA else len(tiles)) // grid
    print(f"\nring tile={tile} stages={stages} grid={grid}: {n_bulk} bulk / {len(tiles)} tiles, {per_cta} per CTA")
    assert per_cta >= 3 * stages, "the ring must wrap around several times in every CTA"
    host = flat.cpu().numpy()
    total = plan.staging_bytes
    img = _image([(off, host[o : o + n]) for off, (o, n) in zip(plan.offsets, segs)], total + GUARD)
    stg = _filled(total + GUARD)
    plan.pack(stg.data_ptr(), _stream())
    torch.cuda.synchronize()
    _assert_bytes(stg, img, "pack")

    # scatter into destinations of the same alignment class: the tile list (and with it the ring) stays the same
    dpos, dend = _same_class_destinations(segs, end)
    dst = _filled(dend + GUARD)
    assert (dst.data_ptr() - flat.data_ptr()) % 16 == 0
    plan.update_ptrs([dst.data_ptr() + d if n else 0 for d, (_, n) in zip(dpos, segs)])
    assert plan.tiles()[0] == n_bulk
    packed = stg.clone()
    plan.scatter(stg.data_ptr(), _stream())
    torch.cuda.synchronize()
    _assert_bytes(dst, _image([(d, host[o : o + n]) for d, (o, n) in zip(dpos, segs)], dst.numel()), "scatter")
    _assert_equal_dev(stg, packed, "scatter source")
    plan.close()


RING_CASES = [(4096, 12, 1), (4096, 12, 4), (8192, 8, 1), (16384, 6, 2), (16384, 12, 1), (32768, 4, 1), (32768, 3, 2), (65536, 3, 1)]


@pytest.mark.parametrize("tile,stages,per_sm", RING_CASES, ids=[f"{t}x{s}x{c}" for t, s, c in RING_CASES])
def test_tma_ring_wraps_around_in_pack_and_scatter(built_library, monkeypatch, tile, stages, per_sm):
    """Stages 12/8/6/4/3 are the five walk_tma instantiations; a stage count is honoured only while it fits the shared-memory
    budget of the launcher (200 KiB), which every case here does."""
    assert stages * tile <= 200 * 1024
    monkeypatch.setenv("NVRX_B200_TMA_STAGES", str(stages))
    monkeypatch.setenv("NVRX_B200_TMA_CTAS_PER_SM", str(per_sm))
    _ring_roundtrip(TMA, tile, stages, _sm_count() * per_sm, seed=tile + stages + per_sm)


def test_ldg_walker_takes_many_tiles_per_cta(built_library, monkeypatch):
    """One CTA per SM: every CTA walks dozens of tiles with the next tile's descriptors prefetched."""
    monkeypatch.setenv("NVRX_B200_LDG_CTAS_PER_SM", "1")
    _ring_roundtrip(LDG, 4096, 12, _sm_count(), seed=7)


# ---------------------------------------------------------------------------------------------------------------------
# b. fused exchange packs on local buffers.  This checks addressing only (shard / slot arithmetic, the own copy, rotation,
#    tile order, one smem slot stored N times): the peers are ordinary local allocations standing in for peer-mapped memory.
#    NVLink peer access is tested in test_gpu_multi.py.
# ---------------------------------------------------------------------------------------------------------------------
def _exchange_state(kind):
    g = torch.Generator(device="cuda").manual_seed(11)
    if kind == "narrow":
        base = torch.randn(420_000, device="cuda", generator=g)
        base[:4] = torch.tensor([float("nan"), float("inf"), -0.0, 1e-40], device="cuda")
        ints = torch.randint(-9, 9, (1001,), device="cuda", generator=g, dtype=torch.int64)
        half = torch.randn(3000, device="cuda", generator=g).to(torch.bfloat16)
        return [base[:100_001], ints, base[100_003 : 100_003 + 8193], half, base[120_001 : 120_078],
                base[130_000:], torch.tensor(3.0, device="cuda")], True
    flat = torch.randint(0, 256, (3 << 20,), dtype=torch.uint8, device="cuda", generator=g)
    sizes = [0, 1, 17, 1000, 1024, 4096 + 3, 20_000, 65536 + 5, 100_007, 300_001, 4095, 33, 7777]
    out, cur = [], 0
    for s in sizes:
        for mis in (0, 3, 8, 13):
            cur = _round(cur, 16) + mis
            out.append(flat[cur : cur + s])
            cur += s
    assert cur < flat.numel()
    return out, False


def _peers(n, slot_off, span):
    """n stand-in peer buffers, 512-byte aligned, in one sentinel-filled allocation; (buffer, stride, base addresses)."""
    stride = _round(slot_off + span + GUARD, 512)
    buf = _filled(n * stride)
    return buf, stride, [buf.data_ptr() + j * stride for j in range(n)]


def _sharded_image(img, total, n, shard, stride, slot_off):
    """Peer j holds [j * shard, (j + 1) * shard) of the packed range at slot_off; gaps keep the sentinel."""
    want = np.full(n * stride, SENTINEL, dtype=np.uint8)
    for j in range(n):
        lo, hi = j * shard, min(total, (j + 1) * shard)
        if hi > lo:
            want[j * stride + slot_off : j * stride + slot_off + hi - lo] = img[lo:hi]
    return want


def _check_plain_pack_and_scatter(plan, tensors, narrow, img, total):
    """After a fused pack the same plan packs and scatters plainly again (it leaves sharded mode)."""
    stg = _filled(total + GUARD)
    plan.pack(stg.data_ptr(), _stream())
    torch.cuda.synchronize()
    _assert_bytes(stg, img, "plain pack after a fused one")
    mask = orc.narrow_mask(tensors, narrow)
    want_t = orc.scatter_oracle(img, [t.shape for t in tensors], [t.dtype for t in tensors], plan.offsets, plan.packed_nbytes, mask)
    nbytes = [w.numel() * w.element_size() for w in want_t]
    cur, pos = 0, []
    for t, nb in zip(tensors, nbytes):
        cur = _round(cur, 16) + t.data_ptr() % 16 + 16  # the sources' classes: the bulk tiles stay
        pos.append(cur)
        cur += nb
    dst = _filled(cur + GUARD)
    plan.update_ptrs([dst.data_ptr() + p if nb else 0 for p, nb in zip(pos, nbytes)])
    packed = stg.clone()
    plan.scatter(stg.data_ptr(), _stream())
    torch.cuda.synchronize()
    _assert_bytes(dst, _image([(p, orc.tensor_bytes(w)) for p, w in zip(pos, want_t)], dst.numel()), "plain scatter")
    _assert_equal_dev(stg, packed, "scatter source")


def _cuts_a_tensor(offsets, packed, shard, total):
    return any(o < k < o + n for k in range(shard, total, shard) for o, n in zip(offsets, packed))


@pytest.mark.parametrize("state", ["ragged", "narrow"])
@pytest.mark.parametrize("variant", ["ldg", "tma"])
@pytest.mark.parametrize("n_peers", [1, 2, 3, 7, 16])
def test_pack_sharded_addressing_on_local_buffers(built_library, monkeypatch, state, variant, n_peers):
    tensors, narrow = _exchange_state(state)
    img, total = _packed_image(tensors, narrow)
    exact, _ = orc.shard_bounds(total, n_peers)
    oversized = exact + 8 * 512  # the last non-empty shard is partial, later ones may be empty
    slot_off = 3 * 512
    peers, stride, bases = _peers(n_peers, slot_off, oversized)
    stg = _filled(total + GUARD)
    for interleave in ("1", "0"):
        monkeypatch.setenv("NVRX_B200_SHARD_INTERLEAVE", interleave)  # read when the tile list is built: one plan each
        plan = _plan(tensors, narrow, tile_bytes=4096, variant=VARIANTS[variant])
        offs, packed = plan.offsets, plan.packed_nbytes
        for shard in (exact, oversized):
            if n_peers > 1 and shard == exact:
                assert _cuts_a_tensor(offs, packed, shard, total), "shard edges must fall inside tensors"
            want = torch.from_numpy(_sharded_image(img, total, n_peers, shard, stride, slot_off)).cuda()
            for own in (True, False):
                for rot in range(n_peers):
                    plan.set_shard_rotation(rot)
                    peers.fill_(SENTINEL)
                    stg.fill_(SENTINEL)
                    plan.pack_sharded(stg.data_ptr() if own else None, bases, shard, slot_off, _stream())
                    torch.cuda.synchronize()
                    what = f"interleave={interleave} shard={shard} own={own} rotation={rot}"
                    _assert_equal_dev(peers, want, "peers " + what)
                    if own:
                        _assert_bytes(stg, img, "own copy " + what)
                    else:
                        assert bool((stg == SENTINEL).all()), "staging written without own copy " + what
        _check_plain_pack_and_scatter(plan, tensors, narrow, img, total)
        plan.close()


@pytest.mark.parametrize("state", ["ragged", "narrow"])
@pytest.mark.parametrize("variant", ["ldg", "tma"])
@pytest.mark.parametrize("n_peers", [1, 3, 16])
def test_pack_broadcast_addressing_on_local_buffers(built_library, state, variant, n_peers):
    tensors, narrow = _exchange_state(state)
    img, total = _packed_image(tensors, narrow)
    slot_off = 5 * 512
    peers, stride, bases = _peers(n_peers, slot_off, total)
    want = np.full(n_peers * stride, SENTINEL, dtype=np.uint8)
    for j in range(n_peers):
        want[j * stride + slot_off : j * stride + slot_off + total] = img[:total]
    want = torch.from_numpy(want).cuda()
    plan = _plan(tensors, narrow, tile_bytes=4096, variant=VARIANTS[variant])
    for _ in range(2):
        peers.fill_(SENTINEL)
        plan.pack_broadcast(bases, slot_off, _stream())
        torch.cuda.synchronize()
        _assert_equal_dev(peers, want, "broadcast")
    _check_plain_pack_and_scatter(plan, tensors, narrow, img, total)
    plan.close()


@pytest.mark.parametrize("mode", ["sharded", "broadcast"])
def test_fused_exchange_ring_wraps_around(built_library, monkeypatch, mode):
    """4 KiB tiles, 12 stages, one CTA per SM: each smem slot is stored to several destinations (own copy + shard, or 4
    peers) in one bulk group, and the ring still wraps around in every CTA."""
    monkeypatch.setenv("NVRX_B200_TMA_CTAS_PER_SM", "1")
    monkeypatch.setenv("NVRX_B200_TMA_STAGES", "12")
    tile, stages, n = 4096, 12, 4
    grid = _sm_count()
    rng = np.random.default_rng(21)
    segs, end = _ring_layout(rng, tile, want_bulk=int(3.6 * stages * grid) + 1)
    g = torch.Generator(device="cuda").manual_seed(21)
    flat = torch.randint(0, 256, (end + GUARD,), dtype=torch.uint8, device="cuda", generator=g)
    src = _carve(flat, segs)
    plan = _plan(src, tile_bytes=tile, variant=TMA)
    host = flat.cpu().numpy()
    total = plan.staging_bytes
    img = _image([(off, host[o : o + nb]) for off, (o, nb) in zip(plan.offsets, segs)], total + GUARD)
    slot_off = 512
    if mode == "sharded":
        shard, _ = orc.shard_bounds(total, n)
        n_bulk = plan.tiles(shard)[0]
        peers, stride, bases = _peers(n, slot_off, shard)
        want = _sharded_image(img, total, n, shard, stride, slot_off)
    else:
        n_bulk = plan.tiles()[0]
        peers, stride, bases = _peers(n, slot_off, total)
        want = np.full(n * stride, SENTINEL, dtype=np.uint8)
        for j in range(n):
            want[j * stride + slot_off : j * stride + slot_off + total] = img[:total]
    print(f"\nfused {mode} ring: {n_bulk} bulk tiles, {n_bulk // grid} per CTA")
    assert n_bulk // grid >= 3 * stages
    stg = _filled(total + GUARD)
    if mode == "sharded":
        plan.pack_sharded(stg.data_ptr(), bases, shard, slot_off, _stream())
    else:
        plan.pack_broadcast(bases, slot_off, _stream())
    torch.cuda.synchronize()
    _assert_bytes(peers, want, mode)
    if mode == "sharded":
        _assert_bytes(stg, img, "own copy")
    plan.close()


# ---------------------------------------------------------------------------------------------------------------------
# c. pipelined snapshot (nvrx_snapshot): pack sub-launches per group of copy chunks, copies on a second stream
# ---------------------------------------------------------------------------------------------------------------------
def _expected_launches(total, chunk, growth):
    """The group rule of nvrx_snapshot: chunks of round_up(chunk, 512) bytes (0 or more than the total: one chunk), at most
    256 of them; pack sub-launches cover 1, g, g^2, ... chunks."""
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


def _snapshot_state(layout):
    g = torch.Generator(device="cuda").manual_seed(31)
    if layout == "narrow":
        return _exchange_state("narrow")[0], True, None
    flat = torch.randint(0, 256, (8 << 20,), dtype=torch.uint8, device="cuda", generator=g)
    sizes = [5000, 0, 65536 + 17, 1 << 20, 33, 4096, 300_003, 1024, 777_777, 15, (1 << 20) + 9]
    out, cur = [], 0
    for i, s in enumerate(sizes * 2):
        cur = _round(cur, 16) + (0 if i % 3 else 5)
        out.append(flat[cur : cur + s])
        cur += s
    assert cur < flat.numel()
    offsets = None
    if layout == "container":
        from nvidia_resiliency_ext.checkpointing.b200 import ptzip

        offsets, _ = ptzip.slot_offsets(_nbytes(out))
    return out, False, offsets


@pytest.mark.parametrize("layout", ["ragged", "narrow", "container"])
@pytest.mark.parametrize("variant", ["ldg", "tma"])
def test_pipelined_snapshot_groups_and_chunks(built_library, monkeypatch, layout, variant):
    from nvidia_resiliency_ext.checkpointing.b200 import _cabi
    from nvidia_resiliency_ext.checkpointing.b200.engine import HostBuffer

    tensors, narrow, offsets = _snapshot_state(layout)
    plan = _plan(tensors, narrow, tile_bytes=4096, variant=VARIANTS[variant], staging_offsets=offsets)
    total = plan.staging_bytes
    img, total_o = _packed_image(tensors, narrow, offsets=offsets)
    assert total_o == total
    if offsets is not None:
        assert list(plan.offsets) == list(offsets)
    # about 40 chunks whose edges fall inside tiles (not a multiple of the tile); 512-byte chunks exceed the cap of 256
    cut = _round(total // 40, 4096) + 1536
    mask = orc.narrow_mask(tensors, narrow)
    spans = [(plan.offsets[s] + (o // 2 if mask[s] else o), nb // 2 if mask[s] else nb) for s, nb, o in plan.tiles()[1]]
    assert any(p < k < p + n for p, n in spans for k in range(cut, total, cut)), "chunk edges must cut tiles"
    assert -(-total // 512) > 256
    chunks = [0, 512, cut, total - 1]
    hb = HostBuffer.create(total + GUARD, pin=True, device=_dev())
    host = hb.as_tensor(total + GUARD)
    stg = _filled(total + GUARD)
    drain = torch.cuda.Stream()
    lib = _cabi.lib()
    try:
        for it, (chunk, growth) in enumerate((c, g) for c in chunks for g in (1, 4, 64)):
            monkeypatch.setenv("NVRX_B200_PACK_GROWTH", str(growth))
            stg.fill_(SENTINEL)
            host.fill_(HOST_SENTINEL)
            torch.cuda.synchronize()
            base = (it + 1) << 40
            _cabi.check(lib.nvrx_snapshot(plan._h, stg.data_ptr(), hb.data_ptr, chunk, hb.progress_ptr, base, _stream(),
                                          drain.cuda_stream, None, None), "nvrx_snapshot")
            torch.cuda.synchronize()
            what = f"chunk={chunk} growth={growth}"
            _assert_bytes(stg, img, "staging " + what)
            want_host = img.copy()
            want_host[total:] = HOST_SENTINEL
            _assert_bytes(host.numpy(), want_host, "host " + what)
            assert hb.progress == base + total, what
            assert plan.last_launches() == _expected_launches(total, chunk, growth), what
    finally:
        plan.close()
        del host
        hb.close()


def test_pipelined_snapshot_of_an_empty_plan(built_library):
    from nvidia_resiliency_ext.checkpointing.b200 import _cabi
    from nvidia_resiliency_ext.checkpointing.b200.engine import HostBuffer, Plan

    plan = Plan([], [], None, device=_dev())
    hb = HostBuffer.create(4096, pin=True, device=_dev())
    drain = torch.cuda.Stream()
    try:
        _cabi.check(_cabi.lib().nvrx_snapshot(plan._h, None, hb.data_ptr, 0, hb.progress_ptr, 12345, _stream(), drain.cuda_stream,
                                              None, None), "nvrx_snapshot")
        torch.cuda.synchronize()
        assert hb.progress == 12345
        assert plan.last_launches() == 0 == _expected_launches(0, 0, 4)
    finally:
        plan.close()
        hb.close()


# ---------------------------------------------------------------------------------------------------------------------
# d. a cached plan re-pointed and launched on another stream while its earlier launch is still queued
# ---------------------------------------------------------------------------------------------------------------------
def test_plan_reuse_across_streams_keeps_queued_launches_on_old_tensors(built_library):
    """Pack on stream A (queued behind a bounded spin), re-point the plan at new tensors of the same sizes and alignment
    class (so only the segment table is re-uploaded) and scatter on stream B.  The upload for B must wait for A's pack on
    the device: A still packs the old tensors.  Every address stays valid either way; a missing wait gives wrong bytes."""
    g = torch.Generator(device="cuda").manual_seed(41)
    segs, cur = [], 0
    for i, s in enumerate([300_000, 17, 65536, 1 << 20, 4097, 250_001, 1000] * 4):
        cur = _round(cur, 16) + (i % 4) * 3
        segs.append((cur, s))
        cur += s
    old_flat = torch.randint(0, 256, (cur + GUARD,), dtype=torch.uint8, device="cuda", generator=g)
    new_flat = _filled(cur + GUARD, 0)
    old, new = _carve(old_flat, segs), _carve(new_flat, segs)
    assert (new_flat.data_ptr() - old_flat.data_ptr()) % 16 == 0
    old_host = old_flat.cpu().numpy()
    plan = _plan(old, tile_bytes=32768)
    n_bulk = plan.tiles()[0]
    total = plan.staging_bytes
    img = _image([(off, old_host[o : o + n]) for off, (o, n) in zip(plan.offsets, segs)], total + GUARD)
    stg_a = _filled(total + GUARD)
    stg_b = torch.randint(0, 256, (total + GUARD,), dtype=torch.uint8, device="cuda", generator=g)
    a, b = torch.cuda.Stream(), torch.cuda.Stream()
    plan.commit(_stream())
    # load both walkers now: a kernel's first launch may load it lazily, and that waits for the whole device (the spin
    # below included), which would order the two streams by accident
    plan.pack(stg_a.data_ptr(), _stream())
    plan.scatter(stg_a.data_ptr(), _stream())  # the old tensors get their own bytes back
    stg_a.fill_(SENTINEL)
    torch.cuda.synchronize()
    _assert_bytes(old_flat, old_host, "old tensors after the warm-up")
    with torch.cuda.stream(a):
        torch.cuda._sleep(200_000_000)  # a bounded spin (~0.1 s) that keeps the pack below queued
    plan.pack(stg_a.data_ptr(), a.cuda_stream)
    plan.update_ptrs(_ptrs(new))
    assert plan.tiles()[0] == n_bulk  # same class: the tile list is kept, only the segments change
    plan.scatter(stg_b.data_ptr(), b.cuda_stream)
    torch.cuda.synchronize()
    _assert_bytes(stg_a, img, "pack queued on stream A before the re-point")
    sb = stg_b.cpu().numpy()
    _assert_bytes(new_flat, _image([(o, sb[off : off + n]) for off, (o, n) in zip(plan.offsets, segs)], new_flat.numel(), 0),
                  "scatter on stream B")
    _assert_bytes(old_flat, old_host, "old tensors")
    plan.close()


# ---------------------------------------------------------------------------------------------------------------------
# e. box scatter geometry
# ---------------------------------------------------------------------------------------------------------------------
def _run_boxes(boxes, src, dst_len, tile):
    """boxes: (elem, sizes, src_off, src_strides, dst_off, dst_strides); scatter on the GPU and compare with box_copy."""
    from nvidia_resiliency_ext.checkpointing.b200.engine import BoxPlan

    stg = torch.from_numpy(src).cuda()
    dst = _filled(dst_len + GUARD)
    bp = BoxPlan([(e, sz, so, ss, dst.data_ptr() + do, ds) for e, sz, so, ss, do, ds in boxes], src.size, device=_dev(),
                 tile_bytes=tile)
    bp.scatter(stg.data_ptr(), _stream())
    torch.cuda.synchronize()
    want = np.full(dst.numel(), SENTINEL, dtype=np.uint8)
    for e, sz, so, ss, do, ds in boxes:
        box_copy(src, want, e, sz, so, ss, do, ds)
    _assert_bytes(dst, want, "box scatter")
    _assert_bytes(stg, src, "box scatter source")
    return bp


@pytest.mark.parametrize("tile", [4096, 32768, 65536])
@pytest.mark.parametrize("seed", range(12))
def test_box_scatter_random_batches(built_library, seed, tile):
    rng = np.random.default_rng(seed)
    boxes, _, src_bytes, dst_bytes = _random_boxes(rng, int(rng.integers(8, 40)), 0)
    src = rng.integers(0, 256, src_bytes + 1, dtype=np.uint8)
    _run_boxes(boxes, src, dst_bytes, tile).close()


def _extent(sizes, strides, elem):
    return elem * (1 + sum((n - 1) * s for n, s in zip(sizes, strides))) if all(sizes) else 0


HAND_BOXES = [
    (1, [200_000], [1], [1]),  # one 200 000-byte run: byte ranges of a tile, each copied by a whole CTA
    (4, [40, 1000], [1003, 1], [1001, 1]),  # 4000-byte rows: byte ranges at 4 KiB tiles, a warp per row at 32 KiB
    (1, [300, 31], [40, 1], [37, 1]),  # 31-byte rows: a thread per row
    (1, [300, 32], [40, 1], [35, 1]),  # 32-byte rows: a warp per row
    (1, [300, 33], [41, 1], [36, 1]),
    (8, [200, 3], [5, 1], [4, 1]),  # 24-byte rows: 8-byte accesses when both sides allow
    (4, [200, 3], [4, 1], [5, 1]),  # 12-byte rows: 4-byte accesses
    (2, [700, 900], [1, 700], [900, 1]),  # transposed bf16: element-wise, 2048 rows per 4 KiB tile
    (16, [50, 60], [1, 50], [60, 1]),  # transposed 16-byte elements
    (4, [2, 3, 2, 2, 3, 2, 2, 3], _contig_strides([3, 4, 3, 3, 4, 3, 3, 4]), _contig_strides([2, 4, 2, 3, 3, 3, 2, 4])),  # 8 dims
    (4, [5, 1000], [0, 1], [1000, 1]),  # zero-stride source dim: one saved row broadcast into five
]


@pytest.mark.parametrize("res", [(0, 0), (8, 8), (4, 12), (2, 6), (3, 3), (0, 5)], ids=lambda r: f"src{r[0]}-dst{r[1]}")
@pytest.mark.parametrize("tile", [4096, 32768])
def test_box_scatter_hand_made_geometry(built_library, tile, res):
    """Each box starts at the given residues mod 16 of the source and destination: equal residues take the aligned
    vector paths, unequal ones the funnel realignment and the narrower steps of the short-row copy."""
    boxes, cs, cd = [], 0, 0
    for elem, sizes, sst, dstr in HAND_BOXES:
        so, do = _round(cs, 16) + res[0], _round(cd, 16) + res[1]
        boxes.append((elem, sizes, so, sst, do, dstr))
        cs, cd = so + _extent(sizes, sst, elem), do + _extent(sizes, dstr, elem)
    src = np.random.default_rng(tile + res[0] * 16 + res[1]).integers(0, 256, cs, dtype=np.uint8)
    bp = _run_boxes(boxes, src, cd, tile)
    tiles = bp.tiles()
    run = [t for t in tiles if t[0] == 0]
    assert all(t[2] == 1 for t in run) and len(run) == -(-200_000 // tile)
    if tile == 4096:
        assert all(t[2] == 1 for t in tiles if t[0] == 1)  # rows longer than half a tile are cut into byte ranges
        assert max(t[2] for t in tiles if t[0] == 7) == 2048
    bp.close()
