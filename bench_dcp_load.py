"""``python bench_dcp_load.py --gpus 1 --steps K --warmup W [--scale S]``: torch.distributed.checkpoint loads of the C2
state (bench.py's workload), stock ``FileSystemReader`` against ``CachedMetadataFileSystemReader(load_on_engine=True)``, alternating the two, on three layouts:

    same      saved by this process from the CUDA state, loaded into the same layout
    shard0    saved as Shard(0) DTensors by 2 gloo CPU ranks, loaded into full CUDA tensors
    shard1    saved as Shard(1) the same way (every read item is a column box: non-contiguous on the saved side)

Prints one JSON line.  Per layout and arm: wall time to device sync and GB/s; for the engine arm the box-kernel time (CUDA
events around the launches only), its
algorithmic bytes and their share of 3.35 TB/s, the peak staging bytes; and whether every loaded tensor is bit-equal
between the arms.  Checkpoints go to a temporary directory (``/dev/shm`` when writable) and are removed after each layout.

``--saved-dtype`` / ``--target-dtype`` (fp32, bf16, fp16; default ``same``) save the floating tensors of the state in one
dtype and load them into targets of another, so the engine arm converts in the box scatter (algorithmic bytes
(es + ed) x elements) and bit-equality is NaN-aware (NaN positions by isnan, everything else by bits).

``--verify`` adds a third arm, the engine reader with ``verify=True`` (every record checked against its CRC-32 on the
GPU), alternating with the other two.  Per layout it adds the arm's wall time, the CRC kernels' time (CUDA events around
their launches only), the bytes they summed and their share of 3.35 TB/s (reads only: S bytes, not 2 S), the host time
of the verify path (range planning, CRC plans and launches, chaining), the per-run wall times of both engine arms, the
bytes read for the checksum alone and whether the arm's tensors are bit-equal to the stock ones.  Without the flag the JSON is
unchanged."""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parent
for _p in (str(ROOT), str(ROOT / "nvidia-resiliency-ext_b200")):
    if _p not in sys.path:
        sys.path.insert(0, _p)

import torch  # noqa: E402
import torch.distributed.checkpoint as dcp  # noqa: E402

HBM_GBS = 3350.0  # H100 SXM data sheet
DTYPES = {"fp32": torch.float32, "bf16": torch.bfloat16, "fp16": torch.float16}


def _as(dtype_name, t):
    """``t`` in dtype ``dtype_name`` when it is an fp32 / bf16 / fp16 tensor and the name is not ``same``."""
    if dtype_name == "same" or t.dtype not in DTYPES.values():
        return t
    return t.to(DTYPES[dtype_name])


def _flat_state(device, scale):
    from bench import flatten, llama3_8b_shard_state

    sd, _ = llama3_8b_shard_state(device, scale=scale)
    return {f"t{i:04d}": t for i, t in enumerate(flatten(sd))}


def _save_sharded(rank, world, port, root, placement, scale, saved_dtype="same"):
    import torch.distributed as dist
    from torch.distributed.device_mesh import init_device_mesh
    from torch.distributed.tensor import Replicate, Shard, distribute_tensor

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    mesh = init_device_mesh("cpu", (world,))
    sd = {}
    for k, v in _flat_state("cpu", scale).items():
        v = _as(saved_dtype, v)
        pl = Shard(placement) if v.dim() > placement else (Shard(0) if v.dim() else Replicate())
        sd[k] = distribute_tensor(v, mesh, [pl])
    dcp.save(sd, checkpoint_id=root)
    dist.barrier()
    dist.destroy_process_group()


def _card():
    try:
        out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, power = [x.strip() for x in out.split(",")[:2]]
        return name, power
    except Exception:  # noqa: BLE001
        return torch.cuda.get_device_name(0), "unknown"


def _bits_equal(a, b):
    return a.dtype == b.dtype and a.shape == b.shape and (
        a.numel() == 0 or torch.equal(a.contiguous().view(-1).view(torch.uint8), b.contiguous().view(-1).view(torch.uint8)))


def _nan_aware_equal(a, b):
    if a.dtype not in DTYPES.values() or a.dtype != b.dtype or a.shape != b.shape:
        return _bits_equal(a, b)
    na, nb = torch.isnan(a), torch.isnan(b)
    return torch.equal(na, nb) and _bits_equal(torch.where(na, torch.zeros_like(a), a), torch.where(nb, torch.zeros_like(b), b))


def run(args):
    from nvidia_resiliency_ext.checkpointing.async_ckpt.cached_metadata_filesystem_reader import CachedMetadataFileSystemReader
    from nvidia_resiliency_ext.checkpointing.b200.engine import SnapshotEngine

    import torch.multiprocessing as mp

    local = 0
    torch.cuda.set_device(local)

    base = "/dev/shm" if os.access("/dev/shm", os.W_OK) else None
    like = {k: _as(args.saved_dtype, v) for k, v in _flat_state("cuda", args.scale).items()}
    total = sum(t.nbytes for t in like.values())
    cast = args.saved_dtype != "same" or args.target_dtype != "same"
    equal = _nan_aware_equal if cast else _bits_equal
    engine = SnapshotEngine.get(local)
    engine.timing = True  # box-kernel time from CUDA events around every launch
    card, power = _card()
    layouts = {}
    for layout in ("same", "shard0", "shard1"):
        root = tempfile.mkdtemp(dir=base, prefix=f"nvrx_dcp_load_{layout}_")
        try:
            if layout == "same":
                dcp.save(like, checkpoint_id=root)
            else:
                ctx = mp.get_context("spawn")
                port = 29600 + (os.getpid() % 200)
                procs = [ctx.Process(target=_save_sharded, args=(r, 2, port, root, int(layout[-1]), args.scale, args.saved_dtype))
                         for r in range(2)]
                for p in procs:
                    p.start()
                for p in procs:
                    p.join()
                assert all(p.exitcode == 0 for p in procs), [p.exitcode for p in procs]
            arms = ("stock", "engine", "verified") if args.verify else ("stock", "engine")
            outs = {arm: {k: torch.empty_like(_as(args.target_dtype, v)) for k, v in like.items()} for arm in arms}
            times = {arm: [] for arm in arms}
            box_ms, stats, crc_ms, verify_host_ms, vstats = [], None, [], [], None
            for it in range(args.warmup + args.steps):
                for arm in arms:
                    reader = (dcp.FileSystemReader(root) if arm == "stock"
                              else CachedMetadataFileSystemReader(root, load_on_engine=True, verify=arm == "verified"))
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    dcp.load(outs[arm], storage_reader=reader)
                    torch.cuda.synchronize()
                    dt = time.perf_counter() - t0
                    if it >= args.warmup:
                        times[arm].append(dt)
                        if arm == "engine":
                            stats = dict(engine.last_box_load)
                            box_ms.append(stats["box_ms"])
                        if arm == "verified":
                            vstats = dict(engine.last_box_load)
                            crc_ms.append(vstats["crc_ms"])
                            verify_host_ms.append(vstats["verify_host_ms"])
            CachedMetadataFileSystemReader.clear_metadata_cache()
            med = {arm: sorted(v)[len(v) // 2] for arm, v in times.items()}
            kms = sorted(box_ms)[len(box_ms) // 2]
            layouts[layout] = {
                "stock_s": round(med["stock"], 4),
                "stock_GBps": round(total / med["stock"] / 1e9, 3),
                "engine_s": round(med["engine"], 4),
                "engine_GBps": round(total / med["engine"] / 1e9, 3),
                "box_kernel_ms": round(kms, 3),
                "box_algorithmic_bytes": stats["algorithmic_bytes"],
                "box_share_of_3p35TBps": round(stats["algorithmic_bytes"] / (kms * 1e-3) / (HBM_GBS * 1e9), 4) if kms else None,
                "box_batches": stats["batches"],
                "peak_staging_bytes": stats["peak_staging_bytes"],
                "bits_equal": all(equal(outs["stock"][k], outs[arm][k]) for arm in arms[1:] for k in like),
            }
            if args.verify:
                cms = sorted(crc_ms)[len(crc_ms) // 2]
                layouts[layout].update(
                    engine_verified_s=round(med["verified"], 4),
                    engine_s_runs=[round(x, 4) for x in times["engine"]],
                    engine_verified_s_runs=[round(x, 4) for x in times["verified"]],
                    verify_host_ms=round(sorted(verify_host_ms)[len(verify_host_ms) // 2], 3),
                    crc_kernel_ms=round(cms, 3),
                    crc_bytes=vstats["crc_bytes"],
                    crc_share_of_3p35TBps=round(vstats["crc_bytes"] / (cms * 1e-3) / (HBM_GBS * 1e9), 4) if cms else None,
                    verified_records=vstats["verified_records"],
                    unverified_records=vstats["unverified_records"],
                    verify_extra_bytes=vstats["verify_extra_bytes"],
                )
            del outs
        finally:
            shutil.rmtree(root, ignore_errors=True)
    config = {"workload": f"C2 state ({total / 1e9:.2f} GB, scale {args.scale}) through dcp.save / dcp.load",
              "steps": args.steps, "warmup": args.warmup, "staging_budget_bytes": SnapshotEngine.DCP_LOAD_STAGING}
    if cast:
        config.update(saved_dtype=args.saved_dtype, target_dtype=args.target_dtype)
    return {
        "metric": "dcp_load_GBps",
        "value": layouts["same"]["engine_GBps"],
        "unit": "GB/s",
        "config": config,
        "gpu": card,
        "power_limit": power,
        "layouts": layouts,
        "bits_equal": all(v["bits_equal"] for v in layouts.values()),
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1, help="one GPU only (the loads run in this process)")
    ap.add_argument("--steps", type=int, default=3, help="timed loads per layout and arm")
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--scale", type=float, default=1.0, help="shrink the state (numbers at != 1.0 are not C2)")
    ap.add_argument("--saved-dtype", choices=["same", *DTYPES], default="same", help="dtype the float tensors are saved in")
    ap.add_argument("--target-dtype", choices=["same", *DTYPES], default="same", help="dtype of the float targets")
    ap.add_argument("--verify", action="store_true", help="add the engine reader with verify=True as a third arm")
    args = ap.parse_args()
    if args.gpus != 1:
        ap.error("dcp-load runs on one GPU (--gpus 1)")
    if not torch.cuda.is_available():
        raise SystemExit("bench_dcp_load.py needs a CUDA device (the engine load path has no CPU fallback)")
    print(json.dumps(run(args)), flush=True)


if __name__ == "__main__":
    main()
