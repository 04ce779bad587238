"""Generates the golden fixtures in this directory by RUNNING THE REFERENCE (``/root/reference/src``).

Run once in the build container (no GPU needed):  ``python tests/golden/make_golden.py``
The GPU box has no ``/root/reference``; tests only read the committed outputs.

What is produced (all inputs are seeded and stored next to the outputs):
  c1_inputs.pt / c1_reference_async.pt   reference config C1: ``AsyncCallsQueue(persistent=True, cpu_shm_mode=True)``
                                          + ``AsyncRequest(torch.save, (preload_tensors(sd), path))`` (core.py:947,
                                          utils.py:85) -- the file the reference's async path writes
  local_inputs.pt / iter_0000007_0_local.pt
                                          ``LocalCheckpointManager.save(BasicTensorAwareStateDict, 7)`` (base_manager.py:237,
                                          local_manager.py:108): the reference's own local snapshot file
  replication.json                        outputs of the reference's ``parse_group_sequence``, ``retrieve_plan``,
                                          ``find_latest`` coverage rule and file-name template on fixed scenarios
  replicate_2rank.json                    ``CliqueReplicationStrategy.replicate`` run on a 2-rank gloo group: order of
                                          returned ids and sha256 of every returned tensor, per rank
  dcp_inputs.pt / dcp_reference/          ``FileSystemWriterAsync`` + ``save_state_dict_async_plan`` + ``AsyncCallsQueue`` +
                                          ``save_state_dict_async_finalize`` (filesystem_async.py:140, state_dict_saver.py:236,417):
                                          the DCP checkpoint directory the reference's async writer produces (CPU tensors)
  bf16_cases.npz                          fp32 bit patterns and ``x.to(torch.bfloat16)`` bits from PyTorch (CPU)
"""
import hashlib
import json
import os
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
REF_SRC = "/root/reference/src"
assert os.path.isdir(REF_SRC), "the reference tree is needed to (re)generate golden vectors"
sys.path.insert(0, REF_SRC)  # the REFERENCE package, not the mirror

import numpy as np  # noqa: E402
import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402
import torch.multiprocessing as mp  # noqa: E402


def sha(t: torch.Tensor) -> str:
    c = t.detach().cpu().contiguous()
    raw = c.view(-1).view(torch.uint8).numpy().tobytes() if c.numel() else b""
    return hashlib.sha256(str(c.dtype).encode() + str(tuple(c.shape)).encode() + raw).hexdigest()


def c1_state_dict():
    g = torch.Generator().manual_seed(0)
    return {
        "model": {
            "w": torch.randn(64, 33, generator=g),
            "b": torch.randn(33, generator=g).to(torch.bfloat16),
            "emb": torch.randint(-(2**31), 2**31 - 1, (17, 5), generator=g, dtype=torch.int32),
        },
        "optimizer": {
            "state": [
                {"exp_avg": torch.randn(64, 33, generator=g) * 1e-3, "step": torch.tensor(12.0)},
                {"exp_avg": torch.randn(7, generator=g).to(torch.float64), "step": torch.tensor(13.0)},
            ],
            "param_groups": [{"lr": 1e-4, "betas": (0.9, 0.95)}],
        },
        "mask": torch.tensor([True, False, True]),
        "bytes": torch.arange(0, 251, dtype=torch.uint8),
        "empty": torch.empty(0, 4),
        "iteration": 1234,
    }


def local_state_dict():
    g = torch.Generator().manual_seed(7)
    return {
        "model": {"q": torch.randn(16, 8, generator=g), "ln": torch.randn(8, generator=g)},
        "optimizer": {"state": {0: {"exp_avg": torch.randn(16, 8, generator=g), "step": torch.tensor(3.0)}}},
        "rng": [torch.randint(0, 255, (11,), generator=g, dtype=torch.uint8), "not-a-tensor", 5],
    }


def init_single_rank():
    os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
    os.environ.setdefault("MASTER_PORT", "29617")
    dist.init_process_group("gloo", rank=0, world_size=1)


def gen_c1():
    from nvidia_resiliency_ext.checkpointing.async_ckpt.core import AsyncCallsQueue, AsyncRequest
    from nvidia_resiliency_ext.checkpointing.utils import preload_tensors

    sd = c1_state_dict()
    torch.save(sd, os.path.join(HERE, "c1_inputs.pt"))
    out = os.path.join(HERE, "c1_reference_async.pt")
    if os.path.exists(out):
        os.remove(out)
    q = AsyncCallsQueue(persistent=True, cpu_shm_mode=True)
    q.schedule_async_request(AsyncRequest(torch.save, (preload_tensors(sd), out), [], {}))
    q.maybe_finalize_async_calls(blocking=True, no_dist=True)
    q.close()
    assert os.path.exists(out)


def gen_local():
    from nvidia_resiliency_ext.checkpointing.local.basic_state_dict import BasicTensorAwareStateDict
    from nvidia_resiliency_ext.checkpointing.local.ckpt_managers.local_manager import LocalCheckpointManager

    sd = local_state_dict()
    torch.save(sd, os.path.join(HERE, "local_inputs.pt"))
    # the reference class asserts is_cuda in __init__ (basic_state_dict.py:89); there is no GPU here, so the
    # object is built without running __init__ -- every other line of the save path is the reference's own
    tasd = BasicTensorAwareStateDict.__new__(BasicTensorAwareStateDict)
    tasd.state_dict = sd
    tasd._is_hollow = False
    with tempfile.TemporaryDirectory() as tmp:
        mgr = LocalCheckpointManager(tmp)
        mgr.save(tasd, 7, is_async=False)
        assert mgr.find_latest() == 7
        src = mgr._local_ckpt_path_from_id(mgr._ckpt_id(7))
        with open(src, "rb") as f, open(os.path.join(HERE, "iter_0000007_0_local.pt"), "wb") as g:
            g.write(f.read())
        names = {
            "file": src.name,
            "dirty": mgr._local_ckpt_path_from_id(mgr._ckpt_id(7), True).name,
            "regex": mgr._filename_from_template("\\d+", "\\d+", "\\"),
            "glob_all": mgr._filename_from_template("*", "*", "*"),
            "glob_iter": mgr._filename_from_template(12, "*", "*"),
            "to_id": list(mgr._filename_to_id("iter_0000042_3_local.pt")),
        }
    return names


def dcp_state_dict():
    g = torch.Generator().manual_seed(11)
    return {
        "model": {
            "w": torch.randn(33, 17, generator=g),
            "b": torch.arange(7, dtype=torch.int64),
            "h": torch.randn(5, 3, generator=g).to(torch.bfloat16),
            "empty": torch.empty(0, 4),
        },
        "opt": {"step": torch.tensor(3), "lr": 0.125, "name": "adam"},
    }


def gen_dcp():
    import shutil

    from torch.distributed.checkpoint import DefaultSavePlanner

    from nvidia_resiliency_ext.checkpointing.async_ckpt.core import AsyncCallsQueue, AsyncRequest
    from nvidia_resiliency_ext.checkpointing.async_ckpt.filesystem_async import FileSystemWriterAsync
    from nvidia_resiliency_ext.checkpointing.async_ckpt.state_dict_saver import (
        save_state_dict_async_finalize,
        save_state_dict_async_plan,
    )

    sd = dcp_state_dict()
    torch.save(sd, os.path.join(HERE, "dcp_inputs.pt"))
    out = os.path.join(HERE, "dcp_reference")
    shutil.rmtree(out, ignore_errors=True)
    q = AsyncCallsQueue(persistent=True, cpu_shm_mode=True)
    writer = FileSystemWriterAsync(out, thread_count=2)
    ret = save_state_dict_async_plan(sd, writer, None, 0, planner=DefaultSavePlanner())
    save_fn, preload_fn, save_args = writer.get_save_function_and_args()
    q.schedule_async_request(AsyncRequest(save_fn, save_args, [], preload_fn=preload_fn))
    q.maybe_finalize_async_calls(blocking=True, no_dist=True)
    try:
        save_state_dict_async_finalize(*ret)
    except RuntimeError as exc:
        # the reference builds its failure flag on torch.cuda.current_device() (state_dict_saver.py:455-459), which needs a
        # GPU; that line runs AFTER the coordinator has written .metadata, so the checkpoint on disk is complete
        assert "NVIDIA driver" in str(exc), exc
    q.close()
    assert os.path.exists(os.path.join(out, ".metadata"))
    with open(os.path.join(out, "torch_version.txt"), "w") as fh:
        fh.write(torch.__version__)


class _StubGroup:
    """Stands in for GroupWrapper in retrieve_plan: fixed member list, canned all_gather_object result."""

    def __init__(self, ranks, gathered):
        self.ranks = ranks
        self._gathered = gathered

    def all_gather_object(self, obj):
        return self._gathered


def gen_replication(names):
    from nvidia_resiliency_ext.checkpointing.local.ckpt_managers.local_manager import LocalCheckpointManager
    from nvidia_resiliency_ext.checkpointing.local.replication.group_utils import parse_group_sequence
    from nvidia_resiliency_ext.checkpointing.local.replication.strategies import (
        CliqueReplicationStrategy,
        NoReplicasAvailableError,
    )

    out = {"names": names, "groups": [], "plans": [], "find_latest": []}
    for j, f, w in [(1, 2, 2), (1, 8, 8), (2, 2, 8), (4, 2, 8), (8, 2, 32), (2, 4, 16), (1, 1, 4), (3, 2, 12), (8, 2, 16)]:
        out["groups"].append({"J": j, "F": f, "W": w, "groups": [list(g) for g in parse_group_sequence(j, f, w)]})

    def ids(it, owners):
        return [[it, o, ""] for o in owners]

    scenarios = [
        # members, available per rank, wanted per member
        {"members": [0, 1], "avail": {0: ids(5, [0, 1]), 1: ids(5, [0, 1])}, "wanted": [ids(5, [0]), ids(5, [1])]},
        {"members": [0, 1], "avail": {0: [], 1: ids(5, [0, 1])}, "wanted": [ids(5, [0]), ids(5, [1])]},
        {"members": [0, 4], "avail": {0: ids(9, [0, 4]), 4: []}, "wanted": [ids(9, [0]), ids(9, [4])]},
        {
            "members": [0, 1, 2, 3, 4, 5, 6, 7],
            "avail": {r: (ids(3, range(8)) if r not in (2, 5) else []) for r in range(8)},
            "wanted": [ids(3, [r]) for r in range(8)],
        },
        {
            "members": [1, 3, 5, 7],
            "avail": {1: ids(2, [1, 3]), 3: ids(2, [3, 5]), 5: ids(2, [5, 7]), 7: ids(2, [7, 1])},
            "wanted": [ids(2, [3]), ids(2, [7]), ids(2, [1]), ids(2, [5])],
        },
        {"members": [0, 1], "avail": {0: [], 1: []}, "wanted": [ids(1, [0]), ids(1, [1])]},
    ]
    for sc in scenarios:
        avail = {r: [tuple(i) for i in v] for r, v in sc["avail"].items()}
        wanted = [[tuple(i) for i in w] for w in sc["wanted"]]
        strat = CliqueReplicationStrategy.__new__(CliqueReplicationStrategy)
        strat.local_group = _StubGroup(sc["members"], wanted)
        strat.target_device = "cpu"
        try:
            plan = strat.retrieve_plan(avail, wanted[0])
            entries = [[e.sender, e.receiver, list(e.id_)] for e in plan.entries]
            err = None
        except NoReplicasAvailableError as e:
            entries, err = None, str(e)
        out["plans"].append(
            {"members": sc["members"], "avail": {str(k): v for k, v in sc["avail"].items()}, "wanted": sc["wanted"],
             "entries": entries, "error": err}
        )

    # coverage rule of find_latest, exercised through the reference manager with canned gathers
    import nvidia_resiliency_ext.checkpointing.local.ckpt_managers.base_manager as bm

    class _GW:
        gathered = None
        ranks = None

        def all_gather_object(self, obj):
            return _GW.gathered

    orig = bm.GroupWrapper
    bm.GroupWrapper = _GW
    try:
        cases = [
            {"ranks": [0, 1], "gathered": [ids(1, [0]) + ids(2, [0]), ids(1, [1])]},
            {"ranks": [0, 1], "gathered": [ids(1, [0]) + ids(2, [0]), ids(1, [1]) + ids(2, [1])]},
            {"ranks": [0, 1, 2, 3], "gathered": [ids(4, [0, 1]), ids(4, [1, 2]), ids(4, [2]), ids(3, [3])]},
            {"ranks": [0, 1, 2, 3], "gathered": [ids(4, [0, 1]), ids(4, [1, 2]), ids(4, [2, 3]), ids(3, [3])]},
            {"ranks": [0, 1], "gathered": [[], []]},
        ]
        for c in cases:
            _GW.gathered = [[tuple(i) for i in g] for g in c["gathered"]]
            _GW.ranks = c["ranks"]
            with tempfile.TemporaryDirectory() as tmp:
                mgr = LocalCheckpointManager(tmp, repl_strategy=object())  # replication "on": foreign ids count
                c["latest"] = mgr.find_latest()
            out["find_latest"].append(c)
    finally:
        bm.GroupWrapper = orig
    with open(os.path.join(HERE, "replication.json"), "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)


def rank_tensors(rank):
    g = torch.Generator().manual_seed(100 + rank)
    return {
        "a": torch.randn(5 + rank, 3, generator=g),
        "nest": [torch.randint(0, 1000, (4,), generator=g, dtype=torch.int64), {"z": torch.randn(2, generator=g).to(torch.float16)}],
        "tag": f"rank{rank}",
    }


def _replicate_worker(rank, world, port, ret):
    sys.path.insert(0, REF_SRC)
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from nvidia_resiliency_ext.checkpointing.local.basic_state_dict import BasicTensorAwareStateDict
    from nvidia_resiliency_ext.checkpointing.local.replication.strategies import CliqueReplicationStrategy

    tasd = BasicTensorAwareStateDict.__new__(BasicTensorAwareStateDict)
    tasd.state_dict = rank_tensors(rank)
    tasd._is_hollow = False
    strat = CliqueReplicationStrategy(dist.group.WORLD, target_device="cpu")
    got, ids = strat.replicate(tasd, (11, rank, ""))
    ret[rank] = {
        "ids": [list(i) for i in ids],
        "tensors": [[sha(t) for t in sd.tensors] for sd in got],
        "tags": [sd.state_dict["tag"] for sd in got],
        "input_hollow": tasd.is_hollow,
    }
    dist.destroy_process_group()


def gen_replicate():
    world = 2
    with mp.Manager() as m:
        ret = m.dict()
        mp.spawn(_replicate_worker, args=(world, 29631, ret), nprocs=world, join=True)
        out = {str(r): ret[r] for r in range(world)}
    out["inputs"] = {str(r): [sha(t) for t in [v for v in _flat(rank_tensors(r)) if isinstance(v, torch.Tensor)]] for r in range(world)}
    with open(os.path.join(HERE, "replicate_2rank.json"), "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)


def _flat(x):
    it = x.values() if isinstance(x, dict) else x
    for v in it:
        if isinstance(v, (dict, list)):
            yield from _flat(v)
        else:
            yield v


def gen_bf16():
    rng = np.random.default_rng(3)
    special = np.array(
        [0x00000000, 0x80000000, 0x3F800000, 0xBF800000, 0x7F800000, 0xFF800000, 0x7F7FFFFF, 0xFF7FFFFF, 0x00000001,
         0x80000001, 0x00007FFF, 0x00008000, 0x00008001, 0x00017FFF, 0x00018000, 0x3F808000, 0x3F818000, 0x3F807FFF,
         0x3F808001, 0x7F7F8000, 0x7F7F7FFF, 0x007FFFFF, 0x00800000, 0x7FC00000, 0xFFC00000, 0x7F800001, 0x7FFFFFFF],
        dtype=np.uint32,
    )
    bits = np.concatenate([special, rng.integers(0, 2**32, 4096, dtype=np.uint64).astype(np.uint32)])
    x = torch.from_numpy(bits.view(np.float32).copy())
    bf = x.to(torch.bfloat16).view(torch.int16).numpy().view(np.uint16)
    np.savez(os.path.join(HERE, "bf16_cases.npz"), f32_bits=bits, bf16_bits_torch_cpu=bf)


if __name__ == "__main__":
    if sys.argv[1:] == ["dcp"]:  # add the DCP fixture without touching the others
        init_single_rank()
        gen_dcp()
        dist.destroy_process_group()
        sys.exit(0)
    gen_bf16()
    gen_replicate()
    init_single_rank()
    gen_c1()
    names = gen_local()
    gen_replication(names)
    gen_dcp()
    dist.destroy_process_group()
    print("golden fixtures written to", HERE)
