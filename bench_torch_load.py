"""``python bench_torch_load.py [--scale S] [--reps N] [--warmup W]``: loading a ``TorchAsyncCheckpoint.async_save`` file of
the C2 state (bench.py's workload: 16.06 GB of fp32 tensors at ``--scale 1``) from ``/dev/shm`` onto the GPU, four arms
run in alternating order:

    torch_load     torch.load(f, map_location="cuda")
    mmap_cuda      torch.load(f, mmap=True), then .cuda() on every tensor
    engine_new     TorchAsyncCheckpoint.load(f, map_location="cuda")     (new CUDA tensors through the engine)
    engine_into    TorchAsyncCheckpoint.load(f, into=state_dict)         (in place into preallocated CUDA tensors)

The engine's pinned slots are released after the save, so the file is read like a resumed process reads it (not the
resident path).  Prints one JSON line: per arm every run's wall time to device sync, the median and GB/s, and whether every
loaded tensor is bit-equal to the saved state; the scatter kernel's time for ``engine_new`` and the box-scatter time for
``engine_into`` (CUDA events around the launches only) and their share of the median load; the card's name and power
limit, read in the same run.  Writes nothing in the repository."""
import argparse
import json
import os
import shutil
import statistics
import sys
import tempfile
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parent
for _p in (str(ROOT), str(ROOT / "nvidia-resiliency-ext_b200")):
    if _p not in sys.path:
        sys.path.insert(0, _p)

import torch  # noqa: E402

ARMS = ("torch_load", "mmap_cuda", "engine_new", "engine_into")


def _all_equal(got, want):
    from bench_dcp_load import _bits_equal
    from nvidia_resiliency_ext.checkpointing.b200.fastload import tensor_leaves

    gl, wl = tensor_leaves(got), tensor_leaves(want)
    return [p for p, _ in gl] == [p for p, _ in wl] and all(a.is_cuda and _bits_equal(a, b) for (_, a), (_, b) in zip(gl, wl))


def _scatter_ms(engine, path, reps=5):
    """Median time of the scatter kernel a new-tensor load of ``path`` launches, CUDA events around the launch only."""
    from nvidia_resiliency_ext.checkpointing.b200.engine import Event
    from nvidia_resiliency_ext.checkpointing.b200.fastload import plan_archive

    plan = plan_archive(path)
    out = [torch.empty(s.nbytes, dtype=torch.uint8, device="cuda") for s in sorted(plan.storages, key=lambda s: s.file_off)]
    del plan
    p = engine._plan_for(out, [False] * len(out))
    staging = engine._ensure_staging(p.staging_bytes)
    stream = torch.cuda.current_stream().cuda_stream
    p.commit(stream)
    times = []
    for _ in range(reps):
        a, b = Event(engine.device, timing=True), Event(engine.device, timing=True)
        a.record(stream)
        p.scatter(staging.ptr, stream)
        b.record(stream)
        b.synchronize()
        times.append(a.elapsed_ms(b))
    return statistics.median(times)


def run(args):
    from bench import llama3_8b_shard_state
    from bench_dcp_load import _card
    from nvidia_resiliency_ext.checkpointing.async_ckpt.torch_ckpt import TorchAsyncCheckpoint
    from nvidia_resiliency_ext.checkpointing.b200.engine import SnapshotEngine
    from nvidia_resiliency_ext.checkpointing.b200.fastload import replace_tensors, tensor_leaves

    if not torch.cuda.is_available():
        raise SystemExit("bench_torch_load.py needs a CUDA device")
    torch.cuda.set_device(0)
    card, power = _card()
    sd, _ = llama3_8b_shard_state("cuda", scale=args.scale)
    total = sum(t.nbytes for _, t in tensor_leaves(sd))
    engine = SnapshotEngine.get(0)
    engine.timing = True  # box-kernel time of the in-place arm from CUDA events around its launches
    base = "/dev/shm" if os.access("/dev/shm", os.W_OK) else None
    root = tempfile.mkdtemp(dir=base, prefix="nvrx_torch_load_")
    ck = TorchAsyncCheckpoint()
    try:
        path = os.path.join(root, "ckpt.pt")
        ck.async_save(sd, path)
        ck.finalize_async_save(blocking=True)
        engine.trim()  # release the slots: the file is read as a restarted process reads it
        into = {"model": {k: torch.zeros_like(v) for k, v in sd["model"].items()},
                "optimizer": {"state": {i: {k: torch.zeros_like(v) for k, v in st.items()} for i, st in sd["optimizer"]["state"].items()}}}

        def load(arm):
            if arm == "torch_load":
                return torch.load(path, map_location="cuda")
            if arm == "mmap_cuda":
                obj = torch.load(path, mmap=True)
                return replace_tensors(obj, {id(t): t.cuda() for _, t in tensor_leaves(obj)})
            if arm == "engine_new":
                return ck.load(path, map_location="cuda")
            ck.load(path, into=into)
            return into

        times = {arm: [] for arm in ARMS}
        equal = {arm: True for arm in ARMS}
        box_ms, stats = [], {}
        for it in range(args.warmup + args.reps):
            order = ARMS if it % 2 == 0 else ARMS[::-1]
            for arm in order:
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                got = load(arm)
                torch.cuda.synchronize()
                dt = time.perf_counter() - t0
                if it >= args.warmup:
                    times[arm].append(dt)
                    if arm == "engine_into":
                        box_ms.append(engine.last_box_load["box_ms"])
                    if arm.startswith("engine"):
                        stats[arm] = dict(engine.last_torch_load)
                equal[arm] = equal[arm] and _all_equal(got, sd)
                del got
                torch.cuda.empty_cache()
        scatter_ms = _scatter_ms(engine, path)
    finally:
        ck.close()
        shutil.rmtree(root, ignore_errors=True)
    arms = {}
    for arm in ARMS:
        med = statistics.median(times[arm])
        arms[arm] = {"runs_s": [round(t, 4) for t in times[arm]], "median_s": round(med, 4), "gb_s": round(total / med / 1e9, 2),
                     "bit_equal": equal[arm]}
    for arm, st in stats.items():
        arms[arm]["stats"] = {k: (round(v, 3) if isinstance(v, float) else v) for k, v in st.items()}
    arms["engine_new"]["scatter_ms"] = round(scatter_ms, 3)
    arms["engine_new"]["scatter_share"] = round(scatter_ms / 1e3 / arms["engine_new"]["median_s"], 4)
    box = statistics.median(box_ms)
    arms["engine_into"]["box_ms"] = round(box, 3)
    arms["engine_into"]["box_share"] = round(box / 1e3 / arms["engine_into"]["median_s"], 4)
    print(json.dumps({
        "bench": "torch_load", "scale": args.scale, "bytes": total, "file": "/dev/shm (tmpfs)", "reps": args.reps,
        "warmup": args.warmup, "card": card, "power_limit": power,
        "speedup_engine_new_vs_torch_load": round(arms["torch_load"]["median_s"] / arms["engine_new"]["median_s"], 2),
        "speedup_engine_into_vs_torch_load": round(arms["torch_load"]["median_s"] / arms["engine_into"]["median_s"], 2),
        "arms": arms,
    }))


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--scale", type=float, default=1.0, help="shrink the C2 state (1.0 = 16.06 GB)")
    ap.add_argument("--reps", type=int, default=3, help="timed loads per arm (the median is reported)")
    ap.add_argument("--warmup", type=int, default=1, help="untimed loads per arm first")
    args = ap.parse_args()
    if args.reps < 3:
        ap.error("--reps must be at least 3")
    run(args)


if __name__ == "__main__":
    main()
