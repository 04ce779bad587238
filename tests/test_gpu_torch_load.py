"""GPU tests of ``TorchAsyncCheckpoint.load`` on the engine: new CUDA tensors equal ``torch.load(f, map_location="cuda")`` in
bytes, dtype, shape, stride, storage offset and storage sharing for every kind of file; in-place loads equal
``target.copy_(saved)`` bit for bit, conversions included, without moving or allocating targets; ``verify=True`` finds one
flipped payload byte; launch counts; the resident read of a file this process just published; a 4.3 GB tensor."""
import gc
import os
import shutil
import uuid

import pytest
import torch

from conftest import GOLDEN
from nvidia_resiliency_ext.checkpointing.async_ckpt.torch_ckpt import TorchAsyncCheckpoint
from nvidia_resiliency_ext.checkpointing.b200 import fastload
from nvidia_resiliency_ext.checkpointing.b200._cabi import SnapError
from nvidia_resiliency_ext.checkpointing.b200.engine import SnapshotEngine

pytestmark = pytest.mark.gpu


@pytest.fixture
def shm_dir():
    d = f"/dev/shm/nvrx_torch_load_{os.getpid()}_{uuid.uuid4().hex[:8]}"
    os.makedirs(d)
    yield d
    shutil.rmtree(d, ignore_errors=True)


def _state(device="cuda"):
    g = torch.Generator(device=device).manual_seed(5)
    base = torch.randn(100_003, device=device, generator=g)
    m = torch.randn(300, 257, device=device, generator=g)
    return {
        "model": {"w": m, "wt": m.t(), "base": base, "view": base[17:90_000:7], "b": torch.randn(4099, device=device, generator=g).to(torch.bfloat16)},
        "optimizer": {"state": {0: {"exp_avg": torch.randn(1000, 33, device=device, generator=g), "step": torch.tensor(7.0, device=device)}}},
        "ids": torch.randint(0, 1 << 40, (333, 7), device=device, generator=g),
        "flags": torch.rand(17, 5, device=device, generator=g) > 0.5,
        "empty": torch.empty(0, 5, device=device),
        "half": torch.randn(64, 48, device=device, generator=g).half(),
        "meta": {"epoch": 3, "name": "run"},
    }


def _bits(t):
    return t.detach().reshape(-1).contiguous().view(torch.uint8) if t.numel() else torch.empty(0, dtype=torch.uint8, device=t.device)


def _assert_same(got, want):
    """Same nested structure, non-tensor leaves, and per tensor device, dtype, shape, stride, storage offset and bytes;
    tensors share a storage exactly where ``want``'s do."""
    gl, wl = fastload.tensor_leaves(got), fastload.tensor_leaves(want)
    assert [p for p, _ in gl] == [p for p, _ in wl]
    share = {}
    for (p, a), (_, b) in zip(gl, wl):
        assert a.device == b.device and a.dtype == b.dtype, p
        assert a.shape == b.shape and a.stride() == b.stride() and a.storage_offset() == b.storage_offset(), p
        assert type(a) is type(b) and a.requires_grad == b.requires_grad, p
        assert a.untyped_storage().nbytes() == b.untyped_storage().nbytes(), p
        assert torch.equal(_bits(a), _bits(b)), p
        if b.untyped_storage().nbytes():
            share.setdefault(b.untyped_storage().data_ptr(), set()).add(a.untyped_storage().data_ptr())
    assert all(len(v) == 1 for v in share.values())
    assert len({next(iter(v)) for v in share.values()}) == len(share)
    strip = lambda x: fastload.replace_tensors(x, {id(t): None for _, t in fastload.tensor_leaves(x)})  # noqa: E731
    assert strip(got) == strip(want)


def _check_new(ck, path, verify=False):
    want = torch.load(path, map_location="cuda")
    got = ck.load(path, map_location="cuda", verify=verify)
    torch.cuda.synchronize()
    _assert_same(got, want)
    stats = SnapshotEngine.get().last_torch_load
    assert stats["mode"] == "new" and stats["entries"] == len(fastload.tensor_leaves(want))
    return stats


@pytest.fixture
def ck():
    c = TorchAsyncCheckpoint()
    yield c
    c.close()


def test_new_tensors_async_save_hard_linked_and_resident(ck, shm_dir):
    sd = _state()
    path = os.path.join(shm_dir, "ckpt.pt")
    ck.async_save(sd, path)
    ck.finalize_async_save(blocking=True)
    eng = SnapshotEngine.get()
    assert os.stat(path).st_nlink > 1  # published as a hard link to the slot
    resident, files, launches = eng.resident_restores, eng.file_restores, eng.launches
    stats = _check_new(ck, path)
    # the resident path: the slot is read in place, nothing is read from the file
    assert eng.resident_restores == resident + 1 and eng.file_restores == files
    assert stats["resident"] and stats["bytes_read"] == 0 and eng.launches - launches == 1 == stats["launches"]


@pytest.mark.parametrize("verify", [False, True])
def test_new_tensors_async_save_copied(shm_dir, monkeypatch, verify):
    monkeypatch.setenv("NVRX_B200_ZERO_COPY", "0")
    monkeypatch.setenv("NVRX_B200_ZIP_CRC", "1")
    c = TorchAsyncCheckpoint()
    try:
        path = os.path.join(shm_dir, "ckpt.pt")
        c.async_save(_state(), path)
        c.finalize_async_save(blocking=True)
        assert os.stat(path).st_nlink == 1
        eng = SnapshotEngine.get()
        files = eng.file_restores
        stats = _check_new(c, path, verify=verify)
        assert not stats["resident"] and stats["bytes_read"] > 0
        if not verify:
            assert eng.file_restores == files + 1
        assert stats["launches"] == (2 if verify else 1)
    finally:
        c.close()


def test_records_without_crc_are_counted_unverified(shm_dir, monkeypatch):
    monkeypatch.setenv("NVRX_B200_ZERO_COPY", "0")
    monkeypatch.setenv("NVRX_B200_ZIP_CRC", "0")
    c = TorchAsyncCheckpoint()
    try:
        path = os.path.join(shm_dir, "nocrc.pt")
        c.async_save(_state(), path)
        c.finalize_async_save(blocking=True)
        n = sum(1 for s in fastload.plan_archive(path).storages if s.nbytes and not s.crc32)
        assert n > 0
        with pytest.warns(UserWarning, match=f"{n} checkpoint records were loaded without a checksum check") as rec:
            stats = _check_new(c, path, verify=True)
        warned = [w for w in rec if "checksum" in str(w.message)]
        assert len(warned) == 1 and warned[0].filename == __file__  # attributed to the caller of TorchAsyncCheckpoint.load
        assert stats["unverified_records"] == n
    finally:
        c.close()


def test_new_tensors_narrowed_async_save(shm_dir):
    c = TorchAsyncCheckpoint(narrow_fp32_to_bf16=True)
    try:
        path = os.path.join(shm_dir, "narrow.pt")
        c.async_save(_state(), path)
        c.finalize_async_save(blocking=True)
        _check_new(c, path)
        # an fp32 target takes the narrowed bytes back, widened on the device like copy_
        into = {"model": {"w": torch.zeros(300, 257, device="cuda")}}
        c.load(path, into=into, strict=False)
        want = torch.zeros(300, 257, device="cuda").copy_(torch.load(path)["model"]["w"])
        assert torch.equal(_bits(into["model"]["w"]), _bits(want))
    finally:
        c.close()


@pytest.mark.parametrize("verify", [False, True])
def test_new_tensors_plain_torch_save(ck, tmp_path, verify):
    sd = _state()
    sd["model"]["p"] = torch.nn.Parameter(torch.randn(10, device="cuda"))
    path = str(tmp_path / "plain.pt")
    torch.save(sd, path)
    stats = _check_new(ck, path, verify=verify)
    assert stats["launches"] == (2 if verify else 1)
    if verify:
        assert stats["verified_records"] == sum(1 for s in fastload.plan_archive(path).storages if s.nbytes)


def test_new_tensors_reference_golden(ck):
    _check_new(ck, str(GOLDEN / "c1_reference_async.pt"))


def test_new_tensors_other_device_index(ck, tmp_path):
    path = str(tmp_path / "plain.pt")
    torch.save(_state("cpu"), path)
    got = ck.load(path, map_location=torch.device("cuda", 0))
    _assert_same(got, torch.load(path, map_location="cuda:0"))


FLOATS = (torch.float32, torch.bfloat16, torch.float16)


def _float_file(tmp_path):
    g = torch.Generator().manual_seed(9)
    sd = {}
    for src in FLOATS:
        x = (torch.randn(257, 129, generator=g) * 1e3).to(src)
        x.view(-1)[:5] = torch.tensor([float("nan"), float("inf"), -float("inf"), -0.0, 7e4]).to(src)
        sd[str(src).split(".")[1]] = x
    sd["ids"] = torch.arange(4096, dtype=torch.int64).reshape(64, 64)
    path = str(tmp_path / "floats.pt")
    torch.save(sd, path)
    return sd, path


def _equal_as_copy(got, want):
    if got.is_floating_point():
        nan = torch.isnan(got)
        assert torch.equal(nan, torch.isnan(want))
        got, want = got.masked_fill(nan, 0), want.masked_fill(nan, 0)
    assert torch.equal(_bits(got), _bits(want))


@pytest.mark.parametrize("contiguous", [True, False])
def test_in_place_all_float_pairs(ck, tmp_path, contiguous):
    sd, path = _float_file(tmp_path)
    saved = torch.load(path)
    for dst in FLOATS:
        into = {}
        for k, v in saved.items():
            dt = dst if v.is_floating_point() else v.dtype
            if contiguous:
                into[k] = torch.full(v.shape, 3, dtype=dt, device="cuda")
            else:
                into[k] = torch.full((v.shape[1], v.shape[0]), 3, dtype=dt, device="cuda").t()
        ptrs = {k: t.data_ptr() for k, t in into.items()}
        gc.collect()
        torch.cuda.synchronize()
        before = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        res = ck.load(path, into=into)
        torch.cuda.synchronize()
        assert res.missing_keys == [] and res.unexpected_keys == []
        smallest = min(t.numel() * t.element_size() for t in into.values())
        assert torch.cuda.max_memory_allocated() - before < smallest and torch.cuda.memory_allocated() <= before
        assert {k: t.data_ptr() for k, t in into.items()} == ptrs
        for k, v in saved.items():
            _equal_as_copy(into[k], torch.full_like(into[k], 3).copy_(v.cuda()))
        stats = SnapshotEngine.get().last_torch_load
        assert stats["fallbacks"] == 0 and stats["entries"] == len(saved)


def test_in_place_fallbacks(ck, tmp_path):
    sd, path = _float_file(tmp_path)
    into = {
        "float32": torch.zeros(257, 129, dtype=torch.float64, device="cuda"),  # fp32 -> fp64: copy_
        "bfloat16": torch.zeros(257, 129, dtype=torch.bfloat16),  # a CPU target: copy_
        "float16": torch.zeros(257, 129, dtype=torch.float32, device="cuda"),  # on the engine
        "ids": torch.zeros(64, 64, dtype=torch.int32, device="cuda"),  # int64 -> int32: copy_
    }
    ck.load(path, into=into)
    stats = SnapshotEngine.get().last_torch_load
    assert stats["fallbacks"] == 3 and stats["entries"] == 4
    saved = torch.load(path)
    for k, t in into.items():
        _equal_as_copy(t, torch.zeros_like(t).copy_(saved[k].to(t.device)))


def test_in_place_strict(ck, tmp_path):
    sd, path = _float_file(tmp_path)
    into = {"float32": torch.zeros(257, 129, device="cuda"), "extra": torch.zeros(3, device="cuda")}
    with pytest.raises(RuntimeError, match="unexpected keys"):
        ck.load(path, into=into)
    assert torch.count_nonzero(into["float32"]) == 0
    res = ck.load(path, into=into, strict=False)
    assert res.missing_keys == ["extra"] and sorted(res.unexpected_keys) == ["bfloat16", "float16", "ids"]
    _equal_as_copy(into["float32"], sd["float32"].cuda())


@pytest.mark.parametrize("verify", [False, True])
def test_in_place_views_shared_and_expanded_records(ck, tmp_path, verify):
    """Saved layouts a DCP load never has: transposed tensors, strided views at a storage offset, several targets reading
    one record, a stride-0 expanded tensor; plus the 8-dim limit of a box (a 9-dim target is copied with copy_)."""
    g = torch.Generator(device="cuda").manual_seed(11)
    sd = _state()
    sd["expanded"] = torch.randn(1, 5, device="cuda", generator=g).expand(4, 5)
    sd["deep8"] = torch.randn(2, 1, 3, 1, 2, 1, 2, 3, device="cuda", generator=g)
    sd["deep9"] = torch.randn(2, 1, 3, 1, 2, 1, 2, 3, 2, device="cuda", generator=g)
    path = str(tmp_path / "views.pt")
    torch.save(sd, path)
    saved = torch.load(path)
    leaves = fastload.tensor_leaves(saved)
    assert saved["expanded"].stride() == (0, 1) and saved["model"]["view"].storage_offset() == 17
    into = fastload.replace_tensors(saved, {id(t): torch.zeros(t.shape, dtype=t.dtype, device="cuda") for _, t in leaves})
    res = ck.load(path, into=into, verify=verify)
    assert res.missing_keys == [] and res.unexpected_keys == []
    stats = SnapshotEngine.get().last_torch_load
    assert stats["fallbacks"] == 1 and stats["entries"] == len(leaves)
    for (p, t), (_, v) in zip(fastload.tensor_leaves(into), leaves):
        _equal_as_copy(t, torch.zeros_like(t).copy_(v))
    if verify:
        plan = fastload.plan_archive(path)
        boxed = {e.storage for e in plan.entries if e.path != ("deep9",) and plan.storages[e.storage].nbytes}
        assert stats["verified_records"] == len(boxed) and stats["host_records"] == 1


def test_in_place_verify_reads_part_of_a_shared_record(ck, tmp_path):
    """Targets that read only part of a record (a strided view, a transposed tensor) still have the whole record checked:
    a flipped byte outside every loaded element raises, naming the key that read the record."""
    sd = _state()
    path = str(tmp_path / "shared.pt")
    torch.save(sd, path)
    saved = torch.load(path)

    def targets():
        return {"model": {"view": torch.zeros_like(saved["model"]["view"], device="cuda"),
                          "wt": torch.zeros(257, 300, device="cuda")}}

    into = targets()
    res = ck.load(path, into=into, strict=False, verify=True)
    assert res.missing_keys == [] and "model.base" in res.unexpected_keys
    assert SnapshotEngine.get().last_torch_load["verified_records"] == 2
    for k in ("view", "wt"):
        assert torch.equal(_bits(into["model"][k]), _bits(saved["model"][k].cuda()))
    bad = str(tmp_path / "bad_shared.pt")
    shutil.copyfile(path, bad)
    plan = fastload.plan_archive(bad)
    off = plan.storages[next(e.storage for e in plan.entries if e.path == ("model", "base"))].file_off + 4  # element 1
    del plan
    with open(bad, "r+b") as fh:
        fh.seek(off)
        b = fh.read(1)
        fh.seek(off)
        fh.write(bytes([b[0] ^ 0x01]))
    with pytest.raises(SnapError, match=r"crc32 mismatch on .*model\.view in .*bad_shared\.pt at record offset"):
        ck.load(bad, into=targets(), strict=False, verify=True)


def test_in_place_launch_counts(ck, tmp_path, monkeypatch):
    sd, path = _float_file(tmp_path)
    into = {k: torch.zeros(v.shape, dtype=v.dtype, device="cuda") for k, v in sd.items()}
    eng = SnapshotEngine.get()
    for budget_mb, verify in ((2048, False), (2048, True)):
        monkeypatch.setattr(SnapshotEngine, "DCP_LOAD_STAGING", budget_mb << 20)
        launches = eng.launches
        ck.load(path, into=into, verify=verify)
        stats = eng.last_torch_load
        assert stats["batches"] == 1 and stats["launches"] == eng.launches - launches
        assert stats["launches"] == (3 if verify else 1)  # one same-dtype box scatter (+ nvrx_crcx_run's two kernels)
    # a budget below the state: several batches, one box scatter each
    monkeypatch.setattr(SnapshotEngine, "DCP_LOAD_STAGING", 64 << 10)
    ck.load(path, into=into)
    stats = eng.last_torch_load
    assert stats["batches"] > 1 and stats["launches"] == stats["batches"]
    for k, v in sd.items():
        assert torch.equal(_bits(into[k]), _bits(v.cuda()))


def _flip(path, dst, key):
    shutil.copyfile(path, dst)
    plan = fastload.plan_archive(dst)
    e = next(e for e in plan.entries if e.path == (key,))
    off = plan.storages[e.storage].file_off + 1001
    del plan, e
    with open(dst, "r+b") as fh:
        fh.seek(off)
        b = fh.read(1)
        fh.seek(off)
        fh.write(bytes([b[0] ^ 0x40]))
    return off


def test_verify_flipped_byte(ck, tmp_path):
    sd, path = _float_file(tmp_path)
    bad = str(tmp_path / "bad.pt")
    _flip(path, bad, "float16")
    with pytest.raises(SnapError, match=r"crc32 mismatch on .*float16 in .*bad\.pt at record offset"):
        ck.load(bad, map_location="cuda", verify=True)
    into = {k: torch.zeros(v.shape, dtype=v.dtype, device="cuda") for k, v in sd.items()}
    with pytest.raises(SnapError, match=r"crc32 mismatch on .*float16 in .*bad\.pt at record offset"):
        ck.load(bad, into=into, verify=True)
    got = ck.load(bad, map_location="cuda")
    for k, v in sd.items():
        diff = (_bits(got[k]) != _bits(v.cuda())).nonzero().flatten().tolist()
        assert diff == ([1001] if k == "float16" else []), k


def test_large_tensor_both_modes(ck, shm_dir):
    n = (4_300_000_000 // 4) + 3  # 4.3 GB of fp32, past 4 GiB
    x = torch.empty(n, dtype=torch.float32, device="cuda")
    x.view(torch.int32).copy_(torch.arange(n, dtype=torch.int32, device="cuda") * -1640531535)  # Knuth's multiplier, as an int32
    path = os.path.join(shm_dir, "large.pt")
    torch.save({"x": x.cpu(), "tail": torch.arange(5.0)}, path)
    got = ck.load(path, map_location="cuda")
    assert torch.equal(_bits(got["x"]), _bits(x)) and torch.equal(got["tail"].cpu(), torch.arange(5.0))
    del got
    torch.cuda.empty_cache()
    into = {"x": torch.zeros_like(x), "tail": torch.zeros(5, device="cuda")}
    ck.load(path, into=into)
    assert torch.equal(_bits(into["x"]), _bits(x)) and torch.equal(into["tail"].cpu(), torch.arange(5.0))
