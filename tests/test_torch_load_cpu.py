"""CPU tests of ``TorchAsyncCheckpoint.load``'s planning half (``b200/fastload.py``): the archive plan of a ``torch.save`` file
against what ``zipfile`` and ``torch.load`` report, the key matching of in-place loads, which targets take the ``copy_``
path, and that the default mode is plain ``torch.load`` while the engine modes refuse to run without CUDA."""
import collections
import struct
import zipfile

import pytest
import torch

from conftest import GOLDEN
from nvidia_resiliency_ext.checkpointing.b200 import fastload, ptzip
from nvidia_resiliency_ext.checkpointing.b200._cabi import SnapError


def _zip_records(path):
    """{key: (data offset, size, crc)} of the data records, from the local headers zipfile points at."""
    out = {}
    with zipfile.ZipFile(path) as zf, open(path, "rb") as fh:
        for key, info in ptzip._data_records(zf).items():
            fh.seek(info.header_offset)
            hdr = fh.read(30)
            name_len, extra_len = struct.unpack_from("<HH", hdr, 26)
            out[key] = (info.header_offset + 30 + name_len + extra_len, info.file_size, info.CRC)
    return out


def _check_plan(path):
    plan = fastload.plan_archive(path)
    recs = _zip_records(path)
    assert sorted(s.key for s in plan.storages) == sorted(recs)
    for s in plan.storages:
        assert (s.file_off, s.record_len, s.crc32) == recs[s.key]
        assert s.nbytes <= s.record_len
    # every entry read back from the raw file bytes at the planned offset equals what a plain torch.load returns
    raw = open(path, "rb").read()
    loaded = dict(fastload.tensor_leaves(torch.load(path, weights_only=True)))
    assert [e.path for e in plan.entries] == list(loaded)
    for e in plan.entries:
        t = loaded[e.path]
        assert (e.dtype, e.size, e.stride, e.storage_offset) == (t.dtype, tuple(t.shape), tuple(t.stride()), t.storage_offset())
        s = plan.storages[e.storage]
        assert s.nbytes == t.untyped_storage().nbytes()
        if s.nbytes:
            storage = torch.frombuffer(bytearray(raw[s.file_off:s.file_off + s.nbytes]), dtype=torch.uint8).untyped_storage()
            got = torch.empty(0, dtype=e.dtype).set_(storage, e.storage_offset, e.size, e.stride)
            assert torch.equal(got.reshape(-1).contiguous().view(torch.uint8), t.reshape(-1).contiguous().view(torch.uint8)), e.path
    # storage sharing: entries share a plan storage exactly when the plain load's tensors share a storage
    ptrs = {}
    for e in plan.entries:
        if plan.storages[e.storage].nbytes:
            ptrs.setdefault(e.storage, set()).add(loaded[e.path].untyped_storage().data_ptr())
    assert all(len(v) == 1 for v in ptrs.values())
    assert len({next(iter(v)) for v in ptrs.values()}) == len(ptrs)
    return plan


def _views_state():
    g = torch.Generator().manual_seed(0)
    base = torch.randn(1000, generator=g)
    m = torch.randn(64, 48, generator=g)
    return {
        "base": base,
        "view": base[10:500:3],  # strided view of a shared storage
        "again": base[7:9],
        "t": m.t(),  # non-contiguous saved tensor
        "m": m,
        "empty": torch.empty(0),
        "empty2": torch.empty(3, 0, dtype=torch.bfloat16),
        "scalar": torch.tensor(3.5, dtype=torch.float64),
        "bf16": torch.randn(33, generator=g).to(torch.bfloat16),
        "ids": torch.arange(17, dtype=torch.int64),
        "expanded": torch.ones(1, 5).expand(4, 5),
        "nested": collections.OrderedDict(a=[torch.zeros(3), (torch.ones(2, dtype=torch.float16), 7)], b="text"),
        "p": torch.nn.Parameter(torch.ones(6)),
        "n": 12,
    }


def test_plan_plain_save_views_shared_empty(tmp_path):
    path = tmp_path / "x.pt"
    sd = _views_state()
    torch.save(sd, path)
    plan = _check_plan(str(path))
    by = {e.path: e for e in plan.entries}
    assert by[("view",)].storage == by[("base",)].storage == by[("again",)].storage
    assert by[("t",)].storage == by[("m",)].storage and by[("t",)].stride == (1, 48)
    assert by[("view",)].storage_offset == 10 and by[("view",)].stride == (3,)
    assert by[("expanded",)].stride == (0, 1)
    assert plan.storages[by[("empty",)].storage].nbytes == 0
    assert by[("nested", "a", 1, 0)].dtype == torch.float16
    assert len(plan.storages) == 11


def test_plan_many_small_tensors(tmp_path):
    path = tmp_path / "many.pt"
    sd = {f"k{i}": torch.full((1 + i % 5,), float(i)) for i in range(100_000)}
    torch.save(sd, path)
    plan = fastload.plan_archive(str(path))
    recs = _zip_records(str(path))
    assert len(plan.storages) == len(plan.entries) == 100_000
    for s in plan.storages[::997]:
        assert (s.file_off, s.record_len, s.crc32) == recs[s.key]
    for e in plan.entries[::997]:
        i = int(e.path[0][1:])
        assert e.size == (1 + i % 5,) and e.storage_offset == 0


def test_plan_reference_golden_file():
    _check_plan(str(GOLDEN / "c1_reference_async.pt"))


@pytest.mark.parametrize("zip64", [False, True])
def test_plan_ptzip_container(tmp_path, zip64):
    g = torch.Generator().manual_seed(1)
    base = torch.randn(300, generator=g)
    obj = {"a": base, "b": base[5:50], "c": torch.randn(7, 9, generator=g).t(), "d": torch.empty(0), "e": torch.arange(4)}
    path = tmp_path / "container.pt"
    ptzip.save(obj, str(path), locate=lambda ptr, nb: None, force_zip64=zip64)
    plan = _check_plan(str(path))
    assert all(s.crc32 for s in plan.storages if s.nbytes)


def test_plan_rejects_unnamed_file_objects():
    import io

    with pytest.raises(ValueError, match="pass a path"):
        fastload.plan_archive(io.BytesIO(b""))


class _NoEngine:
    """Stands in for the engine in the key-matching tests: the targets are CPU tensors, so nothing reaches it."""

    device = 0
    launches = 0
    last_box_load = None

    def __init__(self):
        self.calls = []

    def load_boxes(self, entries, *, verify=False):
        assert not entries, "CPU targets must take the copy_ path"
        self.calls.append(len(entries))


def _saved(tmp_path):
    sd = {"model": {"w": torch.arange(12.0).reshape(3, 4), "b": torch.ones(4)}, "opt": [torch.full((2,), 5.0)]}
    path = tmp_path / "sd.pt"
    torch.save(sd, path)
    return sd, str(path)


def test_match_keys_strict_and_shapes(tmp_path):
    sd, path = _saved(tmp_path)
    plan = fastload.plan_archive(path)
    into = {"model": {"w": torch.zeros(3, 4), "extra": torch.zeros(1)}, "opt": [torch.zeros(3)]}
    pairs, missing, unexpected, bad = fastload.match_keys(plan, into)
    assert missing == ["model.extra"] and unexpected == ["model.b"]
    assert len(bad) == 1 and "opt.0" in bad[0] and "[2]" in bad[0] and "[3]" in bad[0]
    assert sorted(fastload.key_name(plan.entries[i].path) for i, _ in pairs) == ["model.w", "opt.0"]


def test_strict_raises_before_any_read(tmp_path):
    sd, path = _saved(tmp_path)
    eng = _NoEngine()
    into = {"model": {"w": torch.zeros(3, 4), "extra": torch.zeros(1)}, "opt": [torch.zeros(2)]}
    with pytest.raises(RuntimeError, match=r"(?s)unexpected keys: model\.b.*missing keys: model\.extra"):
        fastload._load_into(fastload.plan_archive(path), eng, into, True, False, 0.0)
    assert eng.calls == [] and torch.count_nonzero(into["model"]["w"]) == 0
    into["opt"] = [torch.zeros(5)]  # a shape mismatch raises with strict=False as well, like load_state_dict
    with pytest.raises(RuntimeError, match="size mismatch for opt.0"):
        fastload._load_into(fastload.plan_archive(path), eng, into, False, False, 0.0)
    assert eng.calls == []


def test_non_strict_returns_keys_and_counts_fallbacks(tmp_path):
    sd, path = _saved(tmp_path)
    eng = _NoEngine()
    into = {"model": {"w": torch.zeros(4, 3).t(), "extra": torch.zeros(1)}, "opt": [torch.zeros(2, dtype=torch.float64)]}
    res = fastload._load_into(fastload.plan_archive(path), eng, into, False, False, 0.0)
    assert res.missing_keys == ["model.extra"] and res.unexpected_keys == ["model.b"]
    assert torch.equal(into["model"]["w"], sd["model"]["w"]) and torch.equal(into["opt"][0], sd["opt"][0].double())
    assert eng.last_torch_load["fallbacks"] == 2 and eng.last_torch_load["entries"] == 2


def test_verify_checks_copy_path_records_on_the_host(tmp_path):
    sd, path = _saved(tmp_path)
    plan = fastload.plan_archive(path)
    off = plan.storages[plan.entries[0].storage].file_off  # model.w's record
    del plan
    with open(path, "r+b") as fh:
        fh.seek(off + 5)
        b = fh.read(1)
        fh.seek(off + 5)
        fh.write(bytes([b[0] ^ 0x10]))
    into = {"model": {"w": torch.zeros(3, 4), "b": torch.zeros(4)}, "opt": [torch.zeros(2)]}
    with pytest.raises(SnapError, match=rf"crc32 mismatch on model\.w in .*sd\.pt at record offset {off}"):
        fastload._load_into(fastload.plan_archive(path), _NoEngine(), into, True, True, 0.0)
    assert torch.count_nonzero(into["model"]["w"]) == 0


@pytest.mark.parametrize(
    "device, dtype, dim, saved, want",
    [
        (torch.device("cuda", 0), torch.float32, 2, torch.float32, True),
        (torch.device("cuda", 0), torch.float32, 2, torch.bfloat16, True),
        (torch.device("cuda", 0), torch.float16, 2, torch.bfloat16, True),
        (torch.device("cuda", 0), torch.bfloat16, 2, torch.float16, True),
        (torch.device("cuda", 0), torch.int64, 2, torch.int64, True),
        (torch.device("cuda", 0), torch.uint8, 0, torch.uint8, True),
        (torch.device("cuda", 0), torch.float32, 8, torch.float32, True),
        (torch.device("cuda", 0), torch.float32, 9, torch.float32, False),  # more dims than a box holds
        (torch.device("cuda", 0), torch.bfloat16, 9, torch.float32, False),
        (torch.device("cuda", 0), torch.float64, 2, torch.float32, False),
        (torch.device("cuda", 0), torch.float32, 2, torch.int64, False),
        (torch.device("cuda", 0), torch.int32, 2, torch.int64, False),
        (torch.device("cuda", 1), torch.float32, 2, torch.float32, False),
        (torch.device("cpu"), torch.float32, 2, torch.float32, False),
    ],
)
def test_fallback_classification(device, dtype, dim, saved, want):
    assert fastload.on_engine(device, dtype, dim, saved, 0) is want


def test_map_location_resolution():
    assert fastload.cuda_device("cuda") == torch.device("cuda") and fastload.cuda_device("cuda").index is None
    assert fastload.cuda_device("cuda:1") == torch.device("cuda", 1)
    assert fastload.cuda_device(torch.device("cuda", 2)) == torch.device("cuda", 2)
    for loc in (None, "cpu", torch.device("cpu"), {"cuda:0": "cpu"}, lambda s, loc: s):
        assert fastload.cuda_device(loc) is None


@pytest.mark.parametrize("holder", ["set", "shared_set", "frozenset"])
def test_plan_rejects_tensors_outside_dicts_lists_tuples(tmp_path, holder):
    x = torch.arange(10.0)
    obj = {"set": {"a": x, "s": {torch.ones(3)}}, "shared_set": {"a": x, "s": {x[1:]}},
           "frozenset": {"a": x, "s": frozenset([x[2:4]])}}[holder]
    path = tmp_path / "odd.pt"
    torch.save(obj, path)
    # (frozenset loads only when the user allowlists it, as weights_only requires)
    with torch.serialization.safe_globals([frozenset]), pytest.raises(ValueError, match="containers other than dicts, lists and tuples"):
        fastload.plan_archive(str(path))


def _unqueued():
    """A ``TorchAsyncCheckpoint`` without ``__init__``: ``load`` needs no writer queue, and constructing one would also set
    the class-level ``async_fn`` for the rest of the process."""
    from nvidia_resiliency_ext.checkpointing.async_ckpt.torch_ckpt import TorchAsyncCheckpoint

    return object.__new__(TorchAsyncCheckpoint)


def test_default_mode_is_plain_torch_load(tmp_path, monkeypatch):
    sd, path = _saved(tmp_path)

    def no_engine(*a, **k):
        raise AssertionError("the engine must not be created")

    monkeypatch.setattr(fastload, "_engine_for", no_engine)
    monkeypatch.setattr(fastload, "plan_archive", no_engine)
    ck = _unqueued()
    for loc in (None, "cpu", torch.device("cpu")):
        got = ck.load(path, map_location=loc)
        assert torch.equal(got["model"]["w"], sd["model"]["w"]) and not got["model"]["w"].is_cuda


def test_engine_modes_raise_without_cuda(tmp_path, monkeypatch):
    sd, path = _saved(tmp_path)
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)  # (the real answer on a machine without a GPU)
    ck = _unqueued()
    for loc in ("cuda", torch.device("cuda"), "cuda:0", torch.device("cuda", 0)):
        with pytest.raises(SnapError):
            ck.load(path, map_location=loc)
    with pytest.raises(SnapError):
        ck.load(path, map_location="cuda:0", verify=True)
    with pytest.raises(SnapError):
        ck.load(path, into={"model": {"w": torch.zeros(3, 4)}})
