"""Time nvrx_xor_reduce alone on one GPU with CUDA events: the parity reduce of a save at clique size F = n + 1 over
fragments of S/n bytes (default n = 7, S = 16 GB), with and without clearing the sources.  Prints one JSON line with the
card's name and power limit read in the same run; algorithmic bytes are (n + 1) x fragment, (2n + 1) x fragment with
clearing, compared with the H100 SXM data-sheet HBM3 bandwidth of 3.35 TB/s.

    python tools/bench_xor_reduce.py [--n 7] [--snapshot-gb 16] [--iters 20] [--out xor_reduce.json]
"""
import argparse
import ctypes as C
import json
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
sys.path[:0] = [str(ROOT), str(ROOT / "nvidia-resiliency-ext_b200")]

HBM_PEAK = 3.35e12


def card() -> dict:
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True)
    name, power, clock = (x.strip() for x in out.stdout.splitlines()[0].split(","))
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=7)
    ap.add_argument("--snapshot-gb", type=float, default=16.0)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out")
    args = ap.parse_args()

    import torch

    from nvidia_resiliency_ext.checkpointing.b200._cabi import check, lib

    assert torch.cuda.is_available(), "the measurement needs a GPU"
    torch.cuda.set_device(0)
    n = args.n
    frag = int(args.snapshot_gb * 1e9) // n // 512 * 512
    srcs = [torch.randint(0, 256, (frag,), dtype=torch.uint8, device="cuda") for _ in range(n)]
    dst = torch.empty(frag, dtype=torch.uint8, device="cuda")
    ptrs = (C.c_void_p * n)(*[s.data_ptr() for s in srcs])
    stream = torch.cuda.current_stream().cuda_stream
    result = {"n": n, "fragment_bytes": frag, "snapshot_bytes": n * frag, **card()}
    for clear in (False, True):
        for _ in range(3):
            check(lib().nvrx_xor_reduce(dst.data_ptr(), ptrs, n, frag, int(clear), stream), "nvrx_xor_reduce")
        start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        start.record()
        for _ in range(args.iters):
            check(lib().nvrx_xor_reduce(dst.data_ptr(), ptrs, n, frag, int(clear), stream), "nvrx_xor_reduce")
        stop.record()
        torch.cuda.synchronize()
        ms = start.elapsed_time(stop) / args.iters
        algo = ((2 * n + 1) if clear else (n + 1)) * frag
        key = "clear" if clear else "keep"
        result[key] = {"ms": round(ms, 3), "algorithmic_bytes": algo, "GB_per_s": round(algo / ms / 1e6, 1),
                       "share_of_3_35_TBps": round(algo / ms * 1e3 / HBM_PEAK, 3)}
    line = json.dumps(result)
    print(line)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(line + "\n")


if __name__ == "__main__":
    main()
