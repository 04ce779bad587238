"""Times the checksum kernel (nvrx_crc_run) on the GPU with CUDA events: both table layouts, C2-shaped extents.

    python tools/crc_bench.py [--gb 16] [--reps 7]
Prints one JSON line per variant: GB/s over the bytes the kernel reads, fraction of the measured HBM peak, and a spot check
of the values against zlib."""
import argparse
import json
import os
import sys
import zlib
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
for p in (str(ROOT), str(ROOT / "nvidia-resiliency-ext_b200")):
    sys.path.insert(0, p)

import torch  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gb", type=float, default=16.0)
    ap.add_argument("--reps", type=int, default=7)
    args = ap.parse_args()
    from bench import llama3_8b_shard_shapes
    from nvidia_resiliency_ext.checkpointing.b200 import ptzip
    from nvidia_resiliency_ext.checkpointing.b200.engine import CrcPlan, finish_crcs

    scale = args.gb / 16.06
    sizes = []
    for _, shp in llama3_8b_shard_shapes():
        n = max(1, int(shp[0] * scale)) * (shp[1] if len(shp) == 2 else 1) * 4
        sizes += [n, n, n, n, 4]
    offsets, span = ptzip.slot_offsets(sizes)
    buf = torch.empty(span + 512, dtype=torch.uint8, device="cuda")
    g = torch.Generator(device="cuda").manual_seed(1)
    step = 1 << 28
    for lo in range(0, buf.numel(), step):  # random payload without a second full-size temporary
        buf[lo : lo + step].copy_(torch.randint(0, 256, (min(step, buf.numel() - lo),), dtype=torch.uint8, device="cuda", generator=g))
    plan = CrcPlan(offsets, sizes, torch.cuda.current_device())
    values = torch.zeros(plan.n_values + 2, dtype=torch.int32).pin_memory()
    ready = torch.zeros(1, dtype=torch.int64).pin_memory()
    stream = torch.cuda.current_stream().cuda_stream
    peak = None
    try:
        peak = json.loads((ROOT / "MEASURED_PEAKS.json").read_text()).get("hbm_gbs")
    except Exception:
        pass
    read_bytes = sum(nb // 512 * 512 for nb in sizes)
    for variant in ("private", "shared"):
        os.environ["NVRX_B200_CRC_VARIANT"] = variant
        for _ in range(2):
            plan.run(buf.data_ptr(), values.data_ptr(), ready.data_ptr(), 1, stream)
        torch.cuda.synchronize()
        times = []
        for r in range(args.reps):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            plan.run(buf.data_ptr(), values.data_ptr(), ready.data_ptr(), 2 + r, stream)
            b.record()
            torch.cuda.synchronize()
            times.append(a.elapsed_time(b))
        ms = sorted(times)[len(times) // 2]
        ok = None
        if span < (3 << 30):  # check against zlib only for small runs (needs a host copy of everything): --gb 2
            whole = buf.cpu().numpy()
            crcs = finish_crcs(offsets, sizes, values.data_ptr(), plan.n_values, whole.ctypes.data)
            ok = all(c == zlib.crc32(whole[o : o + n].tobytes()) for c, o, n in list(zip(crcs, offsets, sizes))[::37])
            del whole
        gbps = read_bytes / ms / 1e6
        print(json.dumps({"kernel": f"crc_chunks[{variant}]", "bytes_read": read_bytes, "ms": round(ms, 3), "GBps": round(gbps, 1),
                          "frac_of_hbm_copy_peak": None if not peak else round(gbps / peak, 3), "note": "read-only kernel; the peak is a read+write copy figure", "values_ok": ok, "n_values": plan.n_values}))
    plan.close()


if __name__ == "__main__":
    main()
