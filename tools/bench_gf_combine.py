"""Time nvrx_gf_combine alone on one GPU with CUDA events, beside nvrx_xor_reduce, in one run:

    save      the parity combine of one save at F = 8, m = 2: 12 exchange slots of S/6 into 2 parity rows (sources kept,
              and cleared as a save runs it)
    decode    the two-loss decode of one stripe: 2 parity rows + 4 data fragments of S/6 into 2 fragments
    xor       nvrx_xor_reduce on the m = 1 shape: 7 fragments of S/7 into 1 (sources kept)

Prints one JSON line with the card's name, power limit and maximum SM clock read in the same run; algorithmic bytes are
(n_src + n_dst) x B, (2 n_src + n_dst) x B with clearing, compared with the H100 SXM data-sheet HBM3 bandwidth of
3.35 TB/s.  ``save_vs_xor_per_source_byte`` is the kept save combine's time per source byte over the XOR reduce's.

    python tools/bench_gf_combine.py [--snapshot-gb 16] [--iters 20] [--out gf_combine.json]
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
    ap.add_argument("--snapshot-gb", type=float, default=16.0)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out")
    args = ap.parse_args()

    import numpy as np
    import torch

    from nvidia_resiliency_ext.checkpointing.b200 import erasure
    from nvidia_resiliency_ext.checkpointing.b200._cabi import check, lib

    assert torch.cuda.is_available(), "the measurement needs a GPU"
    torch.cuda.set_device(0)
    S = int(args.snapshot_gb * 1e9)
    F, m = 8, 2
    code = erasure.StripeLayout(list(range(F)), m)
    k = code.k
    frag = S // k // 512 * 512
    srcs = [torch.randint(0, 256, (frag,), dtype=torch.uint8, device="cuda") for _ in range(m * k)]
    dsts = [torch.empty(frag, dtype=torch.uint8, device="cuda") for _ in range(m)]
    stream = torch.cuda.current_stream().cuda_stream
    L = lib()

    def gf(dst_t, src_t, coef, nbytes, clear):
        coef = np.ascontiguousarray(coef, dtype=np.uint8)
        d = (C.c_void_p * len(dst_t))(*[t.data_ptr() for t in dst_t])
        s = (C.c_void_p * len(src_t))(*[t.data_ptr() for t in src_t])
        c = (C.c_uint8 * coef.size).from_buffer_copy(coef.tobytes())
        return lambda: check(L.nvrx_gf_combine(d, len(dst_t), s, len(src_t), c, nbytes, int(clear), stream), "nvrx_gf_combine")

    def timed(fn):
        for _ in range(args.warmup):
            fn()
        start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        start.record()
        for _ in range(args.iters):
            fn()
        stop.record()
        torch.cuda.synchronize()
        return start.elapsed_time(stop) / args.iters

    def entry(ms, n_src, n_dst, nbytes, clear):
        algo = ((2 * n_src if clear else n_src) + n_dst) * nbytes
        return {"ms": round(ms, 3), "n_src": n_src, "n_dst": n_dst, "bytes_each": nbytes, "algorithmic_bytes": algo,
                "GB_per_s": round(algo / ms / 1e6, 1), "share_of_3_35_TBps": round(algo / ms * 1e3 / HBM_PEAK, 3)}

    result = {"F": F, "m": m, "snapshot_bytes": S, "iters": args.iters, **card()}
    enc = code.encode_matrix()
    result["save_keep"] = entry(timed(gf(dsts, srcs, enc, frag, False)), m * k, m, frag, False)
    result["save_clear"] = entry(timed(gf(dsts, srcs, enc, frag, True)), m * k, m, frag, True)

    step = next(s for s in code.rebuild_plan([0, 1]) if len(s.lost) == 2)
    result["decode"] = entry(timed(gf(dsts, srcs[: len(step.sources)], step.matrix, frag, False)), len(step.sources), 2, frag, False)

    n = F - 1
    xfrag = S // n // 512 * 512  # S/7 < S/6: the first 7 exchange slots hold the XOR reduce's sources
    xptrs = (C.c_void_p * n)(*[t.data_ptr() for t in srcs[:n]])
    xdst = dsts[0]
    ms = timed(lambda: check(L.nvrx_xor_reduce(xdst.data_ptr(), xptrs, n, xfrag, 0, stream), "nvrx_xor_reduce"))
    result["xor_m1"] = entry(ms, n, 1, xfrag, False)
    per_src = lambda e: e["ms"] / (e["n_src"] * e["bytes_each"])
    result["save_vs_xor_per_source_byte"] = round(per_src(result["save_keep"]) / per_src(result["xor_m1"]), 3)
    line = json.dumps(result)
    print(line)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(line + "\n")


if __name__ == "__main__":
    main()
