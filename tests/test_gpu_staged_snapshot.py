"""Staged snapshots on one GPU: a save of the structure the engine saw last is launched range by range while the state is
walked and checked, and falls back to one whole snapshot when a tensor changed after ranges were launched.

The drain chunk is 1 MiB, so the ~50 MB state below is cut into four ranges (1, 4, 16 chunks and the rest).  Every file is
read back with ``torch.load`` and compared byte for byte with host copies of the state taken before the save."""
import pytest
import torch

pytestmark = pytest.mark.gpu

MiB = 1 << 20
CHUNK = 1 * MiB
SIZES = [300_000, 7, 65_536, 1_000_003, 0, 2_500_000, 123_457, 512, 1_300_000, 27 * 37]  # fp32 elements


def make_state(seed: int) -> dict:
    g = torch.Generator(device="cuda").manual_seed(seed)
    model = {f"w{i}": torch.randn(n, device="cuda", generator=g) for i, n in enumerate(SIZES)}
    opt = [{"m": torch.randn(n, device="cuda", generator=g),
            "ids": torch.randint(0, 1 << 30, (n // 3 + 1,), device="cuda", generator=g, dtype=torch.int32)} for n in SIZES]
    return {"model": model, "opt": opt, "step": 5, "rng": torch.arange(3)}  # the host tensor travels as it is


def host_copy(sd: dict, narrow: bool) -> dict:
    from nvidia_resiliency_ext.checkpointing.utils import dict_list_map_outplace

    def leaf(v):
        if isinstance(v, torch.Tensor):
            if v.is_cuda and narrow and v.dtype == torch.float32 and v.numel():
                return v.to(torch.bfloat16).cpu()
            return v.detach().cpu().clone()
        return v

    return dict_list_map_outplace(leaf, sd)


def assert_file(path, want: dict) -> None:
    from nvidia_resiliency_ext.checkpointing.utils import _collect_tensors

    got = torch.load(path, weights_only=False)
    assert got["step"] == want["step"] and list(got["model"]) == list(want["model"]) and len(got["opt"]) == len(want["opt"])
    a, b = [], []
    _collect_tensors(got, a)
    _collect_tensors(want, b)
    assert len(a) == len(b)
    for i, (x, y) in enumerate(zip(a, b)):
        assert x.dtype == y.dtype and x.shape == y.shape, i
        assert torch.equal(x.contiguous().view(-1).view(torch.uint8), y.contiguous().view(-1).view(torch.uint8)), i


def group_launches(nbytes: int, chunk: int, growth: int = 4) -> int:
    """Pack launches nvrx_snapshot makes over ``nbytes`` of staging: chunks of round_up(chunk, 512) (at most 256 of them),
    pack groups of 1, 4, 16, ... chunks."""
    if nbytes == 0:
        return 0
    up = lambda v: -(-v // 512) * 512  # noqa: E731
    chunk = up(nbytes if chunk == 0 or chunk > nbytes else chunk)
    n = -(-nbytes // chunk)
    if n > 256:
        chunk = up(-(-nbytes // 256))
        n = -(-nbytes // chunk)
    count, c, g = 0, 0, 1
    while c < n:
        c, g, count = c + g, g * growth, count + 1
    return count


@pytest.fixture
def engine(monkeypatch, built_library):
    from nvidia_resiliency_ext.checkpointing.b200.engine import SnapshotEngine

    torch.cuda.set_device(0)
    monkeypatch.setenv("NVRX_B200_ZERO_COPY", "0")
    eng = SnapshotEngine(0, drain_chunk=CHUNK)
    monkeypatch.setitem(SnapshotEngine._instances, 0, eng)
    yield eng
    torch.cuda.synchronize()
    eng.close()


@pytest.fixture
def ckpt(engine):
    from nvidia_resiliency_ext.checkpointing.async_ckpt.torch_ckpt import TorchAsyncCheckpoint

    made = []

    def make(**kwargs):
        made.append(TorchAsyncCheckpoint(persistent_queue=False, **kwargs))
        return made[-1]

    yield make
    for c in made:
        c.finalize_async_save(blocking=True)
        c.close()


def staged_launches(engine, sd, narrow: bool) -> int:
    """The per-range group rule summed over the ranges of the plan the engine holds for ``sd``."""
    from nvidia_resiliency_ext.checkpointing.b200.engine import staging_ranges
    from nvidia_resiliency_ext.checkpointing.utils import _collect_tensors

    tensors = []
    _collect_tensors(sd, tensors)
    cuda = [t for t in tensors if t.is_cuda]
    plan = engine._plans[engine._plan_key([t.nbytes for t in cuda], engine._narrow_mask(cuda, narrow) if narrow else None, False)]
    bounds = staging_ranges(plan.offsets, plan.staging_bytes, CHUNK)
    assert len(bounds) - 1 == 4, bounds
    ends = [0] + [plan.offsets[b] for b in bounds[1:-1]] + [plan.staging_bytes]
    return sum(group_launches(e - s, CHUNK) for s, e in zip(ends, ends[1:]))


@pytest.mark.parametrize("narrow", [False, True])
@pytest.mark.parametrize("gpu_crc", ["0", "1"])
def test_staged_files_are_byte_exact(engine, ckpt, shm_dir, monkeypatch, narrow, gpu_crc):
    """The second save repeats the first one's structure: staged, one pack launch per group of each range, and in-place
    writes issued right after ``async_save`` returned do not reach the file."""
    monkeypatch.setenv("NVRX_B200_GPU_CRC", gpu_crc)
    c = ckpt(narrow_fp32_to_bf16=narrow)
    sd = make_state(1)
    c.async_save(sd, shm_dir / "first.pt")  # one whole snapshot: the engine learns the structure
    c.finalize_async_save(blocking=True)
    for k in range(2):
        want = host_copy(sd, narrow)
        before = engine.launches
        c.async_save(sd, shm_dir / f"staged{k}.pt")
        assert engine.launches - before == staged_launches(engine, sd, narrow) + (gpu_crc == "1")
        for t in list(sd["model"].values()) + [d[key] for d in sd["opt"] for key in d]:
            t.add_(1)  # on the training stream, behind the pack
        c.finalize_async_save(blocking=True)
        assert_file(shm_dir / f"staged{k}.pt", want)


def _replace(sd, make):
    sd["opt"][-1]["m"] = make(sd["opt"][-1]["m"])  # a tensor of the last range: checked after the first ranges launched


CHANGES = {
    "replaced": lambda sd: _replace(sd, lambda t: torch.randn_like(t)),
    "moved_class": lambda sd: _replace(sd, lambda t: torch.randn(t.numel() + 4, device="cuda")[1 : t.numel() + 1]),
    "non_contiguous": lambda sd: _replace(sd, lambda t: torch.randn(37, 27, device="cuda").t()),
    "on_host": lambda sd: _replace(sd, lambda t: t.cpu()),
    "resized": lambda sd: _replace(sd, lambda t: torch.randn(t.numel() + 1, device="cuda")),
    "removed": lambda sd: sd["opt"][-1].pop("ids"),
    "added": lambda sd: sd["opt"][-1].__setitem__("extra", torch.randn(1000, device="cuda")),
}


@pytest.mark.parametrize("change", list(CHANGES))
def test_structure_changes_between_saves(engine, ckpt, shm_dir, change):
    """One save per stage; between two saves a tensor is replaced, moved, made non-contiguous or removed.  Whatever the
    staged save launched before it met the change, the file equals the state and the progress word keeps rising."""
    c = ckpt()
    sd = make_state(2)
    progress = []
    for stage in range(4):
        if stage == 2:
            CHANGES[change](sd)
        want = host_copy(sd, False)
        c.async_save(sd, shm_dir / f"s{stage}.pt")
        snap = c._pending[max(c._pending)]
        snap.wait()
        progress.append((snap.slot.buf.name, snap.slot.buf.progress, snap.progress_target))
        c.finalize_async_save(blocking=True)
        assert_file(shm_dir / f"s{stage}.pt", want)
    for buf in {p[0] for p in progress}:  # per host buffer (a slot that had to grow starts a new one)
        mine = [p for p in progress if p[0] == buf]
        assert all(got == target for _, got, target in mine)
        assert all(a[2] < b[2] for a, b in zip(mine, mine[1:]))
