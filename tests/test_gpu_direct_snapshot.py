"""Staging-free saves on one GPU (``TorchAsyncCheckpoint(device_staging=False)``): the copy engines move the live tensors
into the pinned slot on the engine's side stream, one small kernel writes the narrowed and small tensors, and ``fence()``
orders the next write after the copies.

Files are compared byte for byte with clones taken at save time.  The ordering tests hold ``_side`` with the sleep kernel of
tests/test_gpu_handoffs.py and assert that the copies were still pending when the write was enqueued."""
import zipfile

import pytest
import torch

from test_gpu_handoffs import (  # noqa: F401 - cycles_per_ms, engines and ckpts are fixtures
    HOLD_MS, _bytes, assert_open, assert_same, ckpts, cycles_per_ms, engines, hold, queued_after,
)

pytestmark = pytest.mark.gpu

MiB = 1 << 20


def _small():
    from nvidia_resiliency_ext.checkpointing.b200.engine import DIRECT_SMALL_BYTES

    return DIRECT_SMALL_BYTES


def odd_state(seed: int) -> dict:
    """Every source alignment 0-15, sizes around the kernel threshold, empty and 4-byte tensors, the small dtypes, a
    non-contiguous tensor and a host tensor."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    t = _small()
    raw = torch.randint(0, 256, (16 * (3 * t + 3 * MiB + 64),), dtype=torch.uint8, device="cuda", generator=g)
    sd, cur = {}, 0
    for a in range(16):
        for n in (t - 1, t, t + 1, 3 * MiB + 7):
            start = -(-cur // 16) * 16 + a  # disjoint views, so that writing one never changes another
            sd[f"a{a}_{n}"] = raw[start:start + n]
            cur = start + n
    sd["empty"] = torch.empty(0, 5, device="cuda")
    sd["scalar"] = torch.tensor(float(seed) + 0.5, device="cuda")
    for dt in (torch.bfloat16, torch.float16):
        sd[str(dt)] = torch.randn(1237, 513, device="cuda", generator=g).to(dt)
    sd["int8"] = torch.randint(-128, 128, (70_001,), dtype=torch.int8, device="cuda", generator=g)
    sd["bool"] = torch.randint(0, 2, (33_333,), device="cuda", generator=g).bool()
    sd["f8"] = torch.randn(1 << 20, device="cuda", generator=g).to(torch.float8_e4m3fn)
    sd["f32"] = torch.randn(1500, 1001, device="cuda", generator=g)
    sd["norm"] = torch.randn(4096, device="cuda", generator=g)
    sd["transposed"] = torch.randn(900, 1300, device="cuda", generator=g).t()
    sd["host"] = torch.arange(1000, dtype=torch.int64)
    return sd


def clones(sd: dict) -> dict:
    return {k: v.clone() for k, v in sd.items()}


def add_one(sd: dict) -> None:
    for v in sd.values():
        if v.is_cuda and v.numel():
            v.add_(1) if v.dtype not in (torch.bool, torch.float8_e4m3fn) else v.copy_(~v if v.dtype == torch.bool else v.float().add(1).to(v.dtype))


def load(path) -> dict:
    return torch.load(path, weights_only=False, mmap=True)


@pytest.mark.parametrize("zero_copy", ["1", "0"])
def test_files_are_bit_exact(engines, ckpts, shm_dir, monkeypatch, zero_copy):
    monkeypatch.setenv("NVRX_B200_ZERO_COPY", zero_copy)
    eng = engines()
    ckpt = ckpts(device_staging=False)
    for i in range(2):
        sd = odd_state(i)
        if zero_copy == "1":
            del sd["host"]  # a host tensor is not in the slot: such a file is always copied
        want = clones(sd)
        path = shm_dir / f"odd{i}.pt"
        ckpt.async_save(sd, path)
        ckpt.fence()
        add_one(sd)  # the next step's writes, fenced
        ckpt.finalize_async_save(blocking=True)
        with zipfile.ZipFile(path) as zf:
            for name in zf.namelist():
                if not name.endswith("/.pad"):  # a published slot's pad record carries no checksum
                    zf.read(name)  # checks the record's CRC-32
        assert_same(load(path), want, f"zero_copy={zero_copy} save {i}")
        assert (path.stat().st_nlink == 2) == (zero_copy == "1")
    assert eng._staging is None


def test_narrowed_records_equal_to_bfloat16(engines, ckpts, shm_dir):
    eng = engines()
    ckpt = ckpts(device_staging=False, narrow_fp32_to_bf16=True)
    sd = odd_state(5)
    want = {k: (v.to(torch.bfloat16) if v.dtype == torch.float32 and v.is_cuda and v.numel() else v.clone()) for k, v in sd.items()}
    launches = eng.launches
    ckpt.async_save(sd, shm_dir / "narrow.pt")
    ckpt.fence()
    ckpt.finalize_async_save(blocking=True)
    assert eng.launches == launches + 1
    assert_same(load(shm_dir / "narrow.pt"), want, "narrowed")
    assert eng._staging is None


def test_large_tensor(engines, ckpts, shm_dir):
    engines()
    ckpt = ckpts(device_staging=False)
    n = 4_300_000_000
    big = torch.empty(n, dtype=torch.uint8, device="cuda")
    big.view(-1)[: n // 8 * 8].view(torch.int64).copy_(torch.arange(n // 8, device="cuda") * 2654435761)
    big[n // 8 * 8:] = 7
    sd = {"head": torch.arange(3, device="cuda"), "big": big[1:], "tail": torch.ones(5, device="cuda")}
    ckpt.async_save(sd, shm_dir / "big.pt")
    ckpt.fence()
    ckpt.finalize_async_save(blocking=True)
    got = load(shm_dir / "big.pt")
    step = 512 * MiB
    for a in range(0, n - 1, step):
        assert torch.equal(got["big"][a:a + step].cuda(), sd["big"][a:a + step]), a
    assert torch.equal(got["head"].cuda(), sd["head"]) and torch.equal(got["tail"].cuda(), sd["tail"])
    del got, big, sd


def test_no_staging_and_no_device_memory(engines, ckpts, shm_dir):
    eng = engines()
    ckpt = ckpts(device_staging=False)
    g = torch.Generator(device="cuda").manual_seed(3)
    sd = {f"p{i}": torch.randn(64 * MiB, device="cuda", generator=g) for i in range(9)}  # 2.25 GB
    sd["step"] = torch.tensor(3.0, device="cuda")
    ckpt.warmup(sd)
    torch.cuda.synchronize()
    free0, _ = torch.cuda.mem_get_info()
    ckpt.async_save(sd, shm_dir / "big.pt")
    torch.cuda.synchronize()
    free1, _ = torch.cuda.mem_get_info()
    assert eng._staging is None
    assert free0 - free1 < 64 * MiB, (free0 - free1) / MiB
    ckpt.finalize_async_save(blocking=True)


def test_fence_orders_the_write(engines, ckpts, shm_dir, cycles_per_ms):
    eng = engines()
    ckpt = ckpts(device_staging=False)
    sd = odd_state(7)
    ckpt.warmup(sd)
    want = clones(sd)
    hold(eng._side.handle, cycles_per_ms)
    ckpt.async_save(sd, shm_dir / "fenced.pt")
    copies = queued_after(eng._side.handle)
    ckpt.fence()
    add_one(sd)
    assert_open(copies)
    ckpt.finalize_async_save(blocking=True)
    assert_same(load(shm_dir / "fenced.pt"), want, "fenced write")


def test_fence_before_adamw_step(engines, ckpts, shm_dir, cycles_per_ms):
    eng = engines()
    ckpt = ckpts(device_staging=False)
    g = torch.Generator(device="cuda").manual_seed(11)
    params = [torch.nn.Parameter(torch.randn(s, device="cuda", generator=g)) for s in ((2048, 1024), (4096,), (3, 5))]
    opt = torch.optim.AdamW(params, lr=1e-2)
    for p in params:
        p.grad = torch.randn(p.shape, device="cuda", generator=g)
    opt.step()  # creates exp_avg / exp_avg_sq
    sd = {"model": {f"p{i}": p for i, p in enumerate(params)}, "optimizer": opt.state_dict()}
    handle = ckpt.fence_before(opt)
    ckpt.warmup(sd)
    want_model = {k: v.detach().clone() for k, v in sd["model"].items()}
    want_state = {k: {kk: vv.clone() for kk, vv in v.items()} for k, v in sd["optimizer"]["state"].items()}
    hold(eng._side.handle, cycles_per_ms)
    ckpt.async_save(sd, shm_dir / "adamw.pt")
    copies = queued_after(eng._side.handle)
    opt.step()  # the hook fences first
    assert_open(copies)
    ckpt.finalize_async_save(blocking=True)
    handle.remove()
    got = load(shm_dir / "adamw.pt")
    assert_same(got["model"], want_model, "params")
    for k, v in want_state.items():
        assert_same(got["optimizer"]["state"][k], v, f"optimizer state {k}")
    assert not torch.equal(params[0].detach(), want_model["p0"]), "the step did not run"


def test_progress_stays_at_base_while_held(engines, ckpts, shm_dir, cycles_per_ms, monkeypatch):
    monkeypatch.setenv("NVRX_B200_ZERO_COPY", "0")
    eng = engines()
    ckpt = ckpts(device_staging=False)
    sd = odd_state(9)
    ckpt.warmup(sd)
    want = clones(sd)
    hold(eng._side.handle, cycles_per_ms)
    ckpt.async_save(sd, shm_dir / "progress.pt")
    snap = ckpt._pending[max(ckpt._pending)]
    copies = queued_after(eng._side.handle)
    base = snap.progress_target - snap.layout.total_bytes
    seen = snap.slot.buf.progress
    assert_open(copies)
    assert seen == base
    ckpt.fence()
    ckpt.finalize_async_save(blocking=True)
    assert snap.slot.buf.progress >= snap.progress_target
    assert_same(load(shm_dir / "progress.pt"), want, "progress")


def _check_state(seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    sd = {f"w{i}": torch.randn(1 << 20, device="cuda", generator=g) for i in range(5)}
    sd["step"] = torch.tensor(1.0, device="cuda")
    sd["half"] = torch.randn(4097, device="cuda", generator=g).to(torch.bfloat16)
    return sd


def test_check_fence_names_the_written_keys(engines, ckpts, shm_dir, cycles_per_ms):
    """The fence checksums on another stream than the one that writes: the writes on the current stream are not fenced,
    run while the copies are held, and end up in the file."""
    from nvidia_resiliency_ext.checkpointing.b200._cabi import SnapError

    eng = engines()
    ckpt = ckpts(device_staging=False, check_fence=True)
    other = torch.cuda.Stream()
    sd = _check_state(1)
    ckpt.warmup(sd)
    ckpt.async_save(sd, shm_dir / "warm_check.pt")  # the checksum kernels' first launch outside the window
    ckpt.fence()
    ckpt.finalize_async_save(blocking=True)
    hold(eng._side.handle, cycles_per_ms)
    ckpt.async_save(sd, shm_dir / "broken.pt")
    copies = queued_after(eng._side.handle)
    ckpt.fence(other)  # checksums now, on `other`
    hold(torch.cuda.current_stream().cuda_stream, cycles_per_ms, HOLD_MS / 4)  # the writes start after the checksums
    sd["w1"].add_(1)
    sd["step"].add_(1)
    assert_open(copies)
    with pytest.raises(SnapError, match="changed between async_save and fence") as err:
        ckpt.finalize_async_save(blocking=True)
    msg = str(err.value)
    assert "'w1'" in msg and "'step'" in msg and "broken.pt" in msg
    assert all(f"'{k}'" not in msg for k in sd if k not in ("w1", "step"))
    torch.cuda.current_stream().wait_stream(other)


def test_check_fence_passes_with_the_fence(engines, ckpts, shm_dir, cycles_per_ms):
    eng = engines()
    ckpt = ckpts(device_staging=False, check_fence=True)
    sd = _check_state(2)
    ckpt.warmup(sd)
    hold(eng._side.handle, cycles_per_ms)
    ckpt.async_save(sd, shm_dir / "kept.pt")
    copies = queued_after(eng._side.handle)
    want = clones(sd)
    ckpt.fence()
    for v in sd.values():
        v.add_(1)
    assert_open(copies)
    ckpt.finalize_async_save(blocking=True)
    assert ckpt.last_fence_check["checked"] == len(sd) and ckpt.last_fence_check["unchecked"] == 0
    assert_same(load(shm_dir / "kept.pt"), want, "fenced")


def test_check_fence_counts_narrowed_as_unchecked(engines, ckpts, shm_dir):
    engines()
    ckpt = ckpts(device_staging=False, check_fence=True, narrow_fp32_to_bf16=True)
    sd = _check_state(3)
    ckpt.async_save(sd, shm_dir / "n.pt")
    ckpt.fence()
    ckpt.finalize_async_save(blocking=True)
    n_f32 = sum(1 for v in sd.values() if v.dtype == torch.float32)
    assert ckpt.last_fence_check["unchecked"] == n_f32
    assert ckpt.last_fence_check["checked"] == len(sd) - n_f32


class _CallLog:
    """The library with every call recorded by name and arguments (then passed on unchanged)."""

    def __init__(self, real):
        self._real, self.calls = real, []

    def __getattr__(self, name):
        fn = getattr(self._real, name)
        if not name.startswith("nvrx_"):
            return fn

        def call(*args):
            self.calls.append((name, args))
            return fn(*args)

        return call


def _handle(x):
    return x.value if hasattr(x, "value") else x


@pytest.mark.parametrize("small", [True, False])
def test_launches_and_nothing_on_the_training_stream(engines, ckpts, shm_dir, monkeypatch, small):
    """One kernel launch with a small tensor, none without; the training stream gets one event record (and the fence's
    wait), every copy and launch goes to the side stream.  Observed at the C ABI, the only way the engine reaches CUDA."""
    from nvidia_resiliency_ext.checkpointing.b200 import _cabi

    log = _CallLog(_cabi.lib())
    monkeypatch.setattr(_cabi, "_LIB", log)
    eng = engines()
    ckpt = ckpts(device_staging=False)
    g = torch.Generator(device="cuda").manual_seed(4)
    sd = {f"w{i}": torch.randn(1 << 20, device="cuda", generator=g) for i in range(4)}
    if small:
        sd["step"] = torch.tensor(2.0, device="cuda")
    ckpt.warmup(sd)
    want = clones(sd)
    launches = eng.launches
    stream = torch.cuda.Stream()  # a training stream with a handle that no other argument can equal
    stream.wait_stream(torch.cuda.current_stream())
    train = stream.cuda_stream
    log.calls.clear()
    with torch.cuda.stream(stream):
        ckpt.async_save(sd, shm_dir / "l.pt")
        ckpt.fence()
    calls = list(log.calls)
    torch.cuda.current_stream().wait_stream(stream)
    ckpt.finalize_async_save(blocking=True)
    assert eng.launches == launches + (1 if small else 0)
    names = [n for n, _ in calls]
    assert names.count("nvrx_snapshot_direct") == 1
    assert not {"nvrx_pack", "nvrx_snapshot", "nvrx_snapshot_range", "nvrx_drain", "nvrx_plan_commit"} & set(names)
    direct = next(a for n, a in calls if n == "nvrx_snapshot_direct")
    assert _handle(direct[12]) == eng._side.handle and (direct[0] is not None) == small
    on_train = [n for n, a in calls if train in [_handle(x) for x in a]]
    assert on_train == ["nvrx_event_record", "nvrx_stream_wait_event"], on_train
    plan = next(p for p in eng._plans.values() if p.n == len(sd) and "_direct" in p.__dict__)
    kernel = plan.__dict__["_direct"]["kernel"]
    assert (kernel is not None) == small and (not small or kernel.last_launches() == 1)
    assert_same(load(shm_dir / "l.pt"), want, "launches")


def test_direct_then_default_then_load_into(engines, ckpts, shm_dir):
    eng = engines()
    direct = ckpts(device_staging=False)
    assert eng._staging is None
    default = ckpts()
    assert eng._staging is not None  # the default save of the fixture's warm-up needs staging
    eng.trim()
    sd = odd_state(12)
    want1 = clones(sd)
    direct.async_save(sd, shm_dir / "m1.pt")
    direct.fence()
    add_one(sd)
    direct.finalize_async_save(blocking=True)
    assert eng._staging is None
    want2 = clones(sd)
    default.async_save(sd, shm_dir / "m2.pt")
    default.finalize_async_save(blocking=True)
    assert eng._staging is not None
    assert_same(load(shm_dir / "m1.pt"), want1, "direct")
    assert_same(load(shm_dir / "m2.pt"), want2, "default")
    direct.async_save(sd, shm_dir / "m3.pt")  # pending while the load writes: load(into=) fences first
    target = {k: v for k, v in sd.items() if v.is_cuda and k != "transposed"}
    direct.load(shm_dir / "m1.pt", into=target, strict=False)
    direct.finalize_async_save(blocking=True)
    assert_same(load(shm_dir / "m3.pt"), want2, "saved before the load")
    assert_same(target, {k: want1[k] for k in target}, "loaded")
