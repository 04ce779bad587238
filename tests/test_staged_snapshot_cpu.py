"""Staged snapshots without a GPU: the range boundaries on the C2 layout, the ranged pointer update against the planner, and
the engine's staged flow and its fallback through a stand-in device that also implements ``nvrx_snapshot_range``."""
import ctypes as C

import pytest
import torch

from _fake_device import FakeCudaTensor, FakeDeviceLib, _val, fake_device, plain

MiB = 1 << 20


def c2_nbytes():
    """Tensor sizes of the C2 state (bench.py's Llama-3-8B row shard) in ``_collect_tensors`` order: model, then per
    parameter main_param, exp_avg, exp_avg_sq and the 4-byte step."""
    import bench

    params = [4 * int(torch.Size(shape).numel()) for _, shape in bench.llama3_8b_shard_shapes()]
    return params + [nb for p in params for nb in (p, p, p, 4)]


def _plan(nbytes, narrow=False, container=False):
    from nvidia_resiliency_ext.checkpointing.b200 import _cabi
    from nvidia_resiliency_ext.checkpointing.b200.engine import Plan
    from nvidia_resiliency_ext.checkpointing.b200.ptzip import slot_offsets

    flags = [_cabi.SEG_NARROW_F32_BF16 if narrow and nb > 4 else 0 for nb in nbytes]
    offsets = None
    if container:
        offsets, _ = slot_offsets([nb // 2 if f else nb for nb, f in zip(nbytes, flags)])
    ptrs = [(i + 1) << 40 for i in range(len(nbytes))]  # never dereferenced: the planner does not touch CUDA
    return Plan(ptrs, nbytes, flags, device=0, staging_offsets=offsets)


@pytest.mark.parametrize("narrow", [False, True])
@pytest.mark.parametrize("container", [False, True])
def test_range_bounds_on_the_c2_layout(built_library, narrow, container):
    from nvidia_resiliency_ext.checkpointing.b200.engine import staging_ranges

    plan = _plan(c2_nbytes(), narrow, container)
    chunk = 256 * MiB
    bounds = staging_ranges(plan.offsets, plan.staging_bytes, chunk)
    assert bounds[0] == 0 and bounds[-1] == plan.n and bounds == sorted(set(bounds))
    ends = [chunk * e for e in (1, 5, 21, 85)]
    want = [0] + [next(i for i, o in enumerate(plan.offsets) if o >= e) for e in ends if e < plan.staging_bytes] + [plan.n]
    assert bounds == want
    assert len(bounds) - 1 == 4  # 256 MiB, 1 GiB, 4 GiB and the rest of the 8 GB (narrowed) or 16 GB (copied)
    assert bounds[1] <= 32  # the first launch waits for the checks of a few tensors only
    # a plan of one chunk or less is one range
    assert staging_ranges(plan.offsets, plan.staging_bytes, plan.staging_bytes) == [0, plan.n]


def _tiles(plan):
    return plan.tiles()


def test_ranged_pointer_update_against_the_planner(built_library):
    nbytes = [4096, 0, 100_000, 7, 65_536, 12]
    plan = _plan(nbytes)
    moved = [p + (1 << 20) if nb else 0 for p, nb in zip(plan.ptrs, nbytes)]
    assert plan.update_ptrs_range(2, moved[2:4]) and plan.update_ptrs_range(4, moved[4:])
    assert plan.ptrs == plan.ptrs[:2] + moved[2:]
    fresh = _plan(nbytes)
    fresh.update_ptrs(plan.ptrs)
    assert _tiles(plan) == _tiles(fresh)  # same work-list as a plan re-pointed at once
    # another 16-byte alignment class would change the tile list: refused, nothing changed
    before = list(plan.ptrs)
    assert not plan.update_ptrs_range(2, [moved[2] + 4, moved[3]])
    assert plan.ptrs == before
    # bad arguments are errors
    from nvidia_resiliency_ext.checkpointing.b200._cabi import SnapError

    with pytest.raises(SnapError):
        plan.update_ptrs_range(2, [0, moved[3]])  # a non-empty segment needs a pointer
    with pytest.raises(SnapError):
        plan.update_ptrs_range(5, [moved[5], moved[5]])  # past the end


class StagedFakeDeviceLib(FakeDeviceLib):
    """The stand-in device plus ``nvrx_snapshot_range``: packs the range's segments and drains its staging bytes."""

    def nvrx_snapshot_range(self, h, lo, hi, staging, host, chunk, progress, base, pack_stream, side, packed_ev, done):
        p, offs, packed = self._layout(h)
        total = C.c_uint64()
        assert self._real.nvrx_plan_info(h, C.byref(total), None, None) == 0
        first = 0 if lo == 0 else offs[lo]
        last = total.value if hi == len(offs) else offs[hi]
        for i in range(lo, hi):
            if p["nbytes"][i]:
                assert not p["flags"][i] & 1
                C.memmove(_val(staging) + offs[i], p["ptrs"][i], p["nbytes"][i])
        C.memmove(_val(host) + first, _val(staging) + first, last - first)
        word = C.c_uint64.from_address(_val(progress))
        assert base + last >= word.value  # the progress word never goes back
        word.value = base + last
        self.calls.append(("range", lo, hi))
        return 0

    def nvrx_plan_update_ptrs_range(self, h, lo, n, ptrs):
        rc = self._real.nvrx_plan_update_ptrs_range(h, lo, n, ptrs)
        if rc == 0:
            self._plans[_val(h)]["ptrs"][lo : lo + n] = [ptrs[k] or 0 for k in range(n)]
        return rc


def _state(seed):
    g = torch.Generator().manual_seed(seed)
    w = FakeCudaTensor.wrap
    return {
        "model": {f"w{i}": w(torch.randn(n, generator=g)) for i, n in enumerate([3000, 7, 5000, 11, 20_000, 900, 6000])},
        "opt": [{"m": w(torch.randn(4000, generator=g)), "ids": w(torch.arange(50) + seed)} for _ in range(3)],
        "step": seed,
    }


def _host(sd):
    from nvidia_resiliency_ext.checkpointing.utils import dict_list_map_outplace

    return dict_list_map_outplace(lambda v: plain(v).clone() if isinstance(v, torch.Tensor) else v, sd)


def _same(a, b):
    from nvidia_resiliency_ext.checkpointing.utils import _collect_tensors

    x, y = [], []
    _collect_tensors(a, x)
    _collect_tensors(b, y)
    assert len(x) == len(y) and a["step"] == b["step"]
    for s, t in zip(x, y):
        s, t = plain(s), plain(t)
        assert s.dtype == t.dtype and s.shape == t.shape
        assert torch.equal(s.contiguous().view(-1).view(torch.uint8), t.contiguous().view(-1).view(torch.uint8))


CHANGES = {
    "same": lambda sd: None,
    "replaced": lambda sd: sd["opt"][2].__setitem__("m", FakeCudaTensor.wrap(torch.randn(4000))),
    "non_contiguous": lambda sd: sd["opt"][2].__setitem__("m", FakeCudaTensor.wrap(torch.randn(80, 50).t())),
    "resized": lambda sd: sd["opt"][2].__setitem__("m", FakeCudaTensor.wrap(torch.randn(4001))),
    "on_host": lambda sd: sd["opt"][2].__setitem__("m", torch.randn(4000)),
    "removed": lambda sd: sd["opt"][2].pop("ids"),
    "added": lambda sd: sd["opt"][2].__setitem__("x", FakeCudaTensor.wrap(torch.randn(10))),
}


@pytest.mark.parametrize("change", list(CHANGES))
def test_staged_flow_and_fallback(monkeypatch, built_library, shm_dir, dist_1rank, change):
    """Two saves of one structure, then one with ``change`` in the last range: the staged saves launch their ranges one by
    one, the changed one falls back to a whole snapshot after them, and every file loads to what ``torch.save`` of the state loads to."""
    from nvidia_resiliency_ext.checkpointing.async_ckpt.torch_ckpt import TorchAsyncCheckpoint
    from nvidia_resiliency_ext.checkpointing.b200.engine import staging_ranges

    monkeypatch.setenv("NVRX_B200_ZERO_COPY", "0")
    with fake_device(monkeypatch) as (engine, lib):
        lib.__class__ = StagedFakeDeviceLib
        engine.drain_chunk = 4096  # the ~190 KB state spans four ranges
        ckpt = TorchAsyncCheckpoint(persistent_queue=False)
        try:
            sd = _state(0)
            for i in range(3):
                if i == 2:
                    CHANGES[change](sd)
                want = _host(sd)
                lib.calls.clear()
                ckpt.async_save(sd, shm_dir / f"s{i}.pt")
                ranges = [c for c in lib.calls if isinstance(c, tuple)]
                if i == 0:
                    assert not ranges and lib.calls.count("pack") == 1  # the first save learns the structure
                elif i == 1 or change in ("same", "replaced"):
                    plan = next(iter(engine._plans.values()))
                    bounds = staging_ranges(plan.offsets, plan.staging_bytes, engine.drain_chunk)
                    assert len(bounds) >= 4 and ranges == [("range", a, b) for a, b in zip(bounds, bounds[1:])]
                    assert "pack" not in lib.calls
                else:
                    assert ranges and lib.calls.count("pack") == 1  # ranges launched, then the whole snapshot behind them
                ckpt.finalize_async_save(blocking=True)
                expect = shm_dir / f"e{i}.pt"
                torch.save(want, expect)
                _same(torch.load(shm_dir / f"s{i}.pt", weights_only=False), torch.load(expect, weights_only=False))
                _same(torch.load(shm_dir / f"s{i}.pt", weights_only=False), want)
        finally:
            ckpt.close()
