"""``python bench_direct_snapshot.py [--scale S] [--rounds N] [--gemm-ms 50,300,600]``: what a checkpoint of the C2 state
(bench.py's workload: 16.06 GB of fp32 tensors at ``--scale 1``) costs the training stream with device staging (the
default) and staging-free (``TorchAsyncCheckpoint(device_staging=False)``), the two arms alternating in one process.

A training step is a loop of bf16 GEMMs lasting about G ms (forward and backward: they only read the state), then
``fence()``, then one ``torch._foreach_add_`` over every state tensor (the optimizer step).  A round times two steps
without a checkpoint, then a step that ends with ``async_save`` and the step after it, with CUDA events on the training
stream; the checkpoint's added time is the second pair minus the first.  Per arm and G it reports the medians of:

    save_host_ms      host time of the async_save call
    added_ms          training-stream time the checkpoint adds over the two steps it touches
    fence_ms          training-stream time from before fence() to after it (its GPU wait)
    to_host_ms, GBps  from the save's position on the training stream to the end of the copies on the side stream
    extra_device_MiB  device memory the arm's first save allocated (torch.cuda.mem_get_info)

It also times the choice of the staging-free kernel threshold: 256 tensors of one size moved all by copy-engine D2H
copies or all by the small pack kernel, per size.  The last file of each arm is compared bit for bit with the state at its
save.  The card's name and power limit are read in the same run.  Files go to a temporary directory on /dev/shm; nothing
is written in the repository."""
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

MiB = 1 << 20


def gemm_loop(ms: float, a: torch.Tensor, per_ms: float) -> None:
    for _ in range(max(1, round(ms * per_ms))):
        torch.mm(a, a)


def gemms_per_ms(a: torch.Tensor) -> float:
    gemm_loop(0, a, 1)
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(200):
        torch.mm(a, a)
    e.record()
    e.synchronize()
    return 200 / s.elapsed_time(e)


def threshold_sweep(engine, sizes=(4, 2048, 16 << 10, 64 << 10, 256 << 10, 1 << 20), n=256):
    """Device time (start event -> end of the side stream's work) of one staging-free snapshot of n tensors of each size,
    moved all by copies (threshold 0) or all by the kernel (threshold above the size)."""
    from nvidia_resiliency_ext.checkpointing.b200 import engine as eng_mod

    side = torch.cuda.ExternalStream(engine._side.handle)
    out = {}
    keep = eng_mod.DIRECT_SMALL_BYTES
    try:
        for size in sizes:
            tensors = [torch.randint(0, 255, (size,), dtype=torch.uint8, device="cuda") for _ in range(n)]
            row = {}
            for label, small in (("copies_us", 0), ("kernel_us", size + 1)):
                eng_mod.DIRECT_SMALL_BYTES = small
                times = []
                for rep in range(6):
                    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    torch.cuda.synchronize()
                    s.record()
                    snap = engine.snapshot(tensors, container=False, direct=True)
                    e.record(side)
                    e.synchronize()
                    snap.release()
                    if rep:
                        times.append(s.elapsed_time(e) * 1e3)
                row[label] = round(statistics.median(times), 1)
            out[size] = row
    finally:
        eng_mod.DIRECT_SMALL_BYTES = keep
    return out


def state_tensors(sd):
    return [t for st in (sd["model"].values(), *[d.values() for d in sd["optimizer"]["state"].values()]) for t in st]


def run_arm(direct, sd, tensors, gemm_ms, rounds, root, a, per_ms, engine):
    from nvidia_resiliency_ext.checkpointing.async_ckpt.torch_ckpt import TorchAsyncCheckpoint

    ck = TorchAsyncCheckpoint(persistent_queue=False, device_staging=not direct)
    side = torch.cuda.ExternalStream(engine._side.handle)
    path = os.path.join(root, f"{'direct' if direct else 'staged'}.pt")
    res = {k: [] for k in ("save_host_ms", "added_ms", "fence_ms", "to_host_ms")}
    extra = None
    total = sum(t.nbytes for t in tensors)
    snap_clone = None

    def step(save_path=None):
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
        ev[0].record()
        gemm_loop(gemm_ms, a, per_ms)
        ev[1].record()
        ck.fence()
        ev[2].record()
        torch._foreach_add_(tensors, 1.0)
        host_ms = copy = None
        if save_path is not None:
            c0 = torch.cuda.Event(enable_timing=True)
            c0.record()
            t0 = time.perf_counter()
            ck.async_save(sd, save_path)
            host_ms = (time.perf_counter() - t0) * 1e3
            c1 = torch.cuda.Event(enable_timing=True)
            c1.record(side)
            copy = (c0, c1)
        ev[3].record()
        return ev, host_ms, copy

    try:
        warm = 2  # slots (a published file keeps one until it is replaced), plans, first launches
        for r in range(rounds + warm):
            free0 = torch.cuda.mem_get_info()[0]
            torch.cuda.synchronize()
            base = [step(), step()]
            saved = step(path)
            if r == rounds + warm - 1:
                snap_clone = [t.clone() for t in tensors]  # the state the file must hold; outside the timed steps
            follow = step()
            torch.cuda.synchronize()
            free1 = torch.cuda.mem_get_info()[0]
            if extra is None:
                extra = (free0 - free1) / MiB
            ck.finalize_async_save(blocking=True)
            print(f"{'direct' if direct else 'staged'} G={gemm_ms:g} round {r}", file=sys.stderr, flush=True)
            if r < warm:
                continue
            el = lambda s: s[0][0].elapsed_time(s[0][3])  # noqa: E731
            res["added_ms"].append(el(saved) + el(follow) - el(base[0]) - el(base[1]))
            res["fence_ms"].append(follow[0][1].elapsed_time(follow[0][2]))
            res["save_host_ms"].append(saved[1])
            res["to_host_ms"].append(saved[2][0].elapsed_time(saved[2][1]))
        got = torch.load(path, mmap=True, weights_only=True)
        got_t = state_tensors(got)
        raw = lambda t: t.reshape(-1).view(torch.uint8)  # noqa: E731 - bytes: the state holds NaN
        bit_equal = all(torch.equal(raw(g.cuda()), raw(w)) for g, w in zip(got_t, snap_clone))
        os.unlink(path)
    finally:
        ck.close()
        snap_clone = None
    med = {k: round(statistics.median(v), 3) for k, v in res.items()}
    med["GBps"] = round(total / (med["to_host_ms"] * 1e-3) / 1e9, 2)
    med["extra_device_MiB"] = round(extra, 1)
    med["bit_equal"] = bit_equal
    med["all"] = {k: [round(x, 3) for x in v] for k, v in res.items()}
    return med


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scale", type=float, default=1.0)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--gemm-ms", default="50,300,600")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_direct_snapshot.py needs a CUDA device")
    from bench import llama3_8b_shard_state
    from bench_dcp_load import _card
    from nvidia_resiliency_ext.checkpointing.b200.engine import DIRECT_SMALL_BYTES, SnapshotEngine

    torch.cuda.set_device(0)
    card, power = _card()
    engine = SnapshotEngine.get(0)
    sweep = threshold_sweep(engine)
    print(f"threshold sweep {sweep}", file=sys.stderr, flush=True)
    engine.trim()
    sd, _ = llama3_8b_shard_state("cuda", scale=args.scale)
    tensors = state_tensors(sd)
    a = torch.randn(8192, 8192, device="cuda", dtype=torch.bfloat16)
    per_ms = gemms_per_ms(a)
    base = "/dev/shm" if os.access("/dev/shm", os.W_OK) else None
    root = tempfile.mkdtemp(dir=base, prefix="nvrx_direct_")
    small = sum(1 for t in tensors if t.nbytes < DIRECT_SMALL_BYTES)
    out = {"bench": "direct_snapshot", "scale": args.scale, "bytes": sum(t.nbytes for t in tensors), "tensors": len(tensors),
           "kernel_tensors": small, "copies": len(tensors) - small, "threshold_bytes": DIRECT_SMALL_BYTES,
           "card": card, "power_limit": power, "gemms_per_ms": round(per_ms, 3), "threshold_sweep_us": sweep, "arms": {}}
    try:
        for g in (float(x) for x in args.gemm_ms.split(",")):
            for direct in (True, False):  # alternating; the staging-free arm first, before any staging exists
                out["arms"][f"{'direct' if direct else 'staged'}_G{int(g)}"] = run_arm(
                    direct, sd, tensors, g, args.rounds, root, a, per_ms, engine)
    finally:
        shutil.rmtree(root, ignore_errors=True)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
