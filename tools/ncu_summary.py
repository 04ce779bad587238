"""Summarise an `ncu --set full` report of the walkers into profiles/<name>.json + .md (run in the build container):

    python tools/ncu_summary.py prof_walk.ncu-rep ncu_walk_summary --commit <sha> \
        --labels "pack TMA walker (C2 bit copy)" "scatter TMA walker" "pack LDG walker" "scatter LDG walker" \
                 "pack LDG narrow fp32->bf16 (C3)" "scatter LDG widen bf16->fp32"
"""
import argparse
import csv
import io
import json
import subprocess

KEEP = [
    "gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum", "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed",
    "dram__throughput.avg.pct_of_peak_sustained_elapsed", "sm__warps_active.avg.pct_of_peak_sustained_active", "launch__registers_per_thread",
    "launch__grid_size", "launch__block_size", "launch__shared_mem_per_block_dynamic", "sm__throughput.avg.pct_of_peak_sustained_elapsed",
    "l1tex__t_sectors_pipe_lsu_mem_global_op_ld.sum", "l1tex__t_sectors_pipe_lsu_mem_global_op_st.sum",
    "lts__t_sectors_srcunit_tex_op_read.sum", "lts__t_sectors_srcunit_tex_op_write.sum", "smsp__inst_executed.sum",
    "launch__occupancy_limit_shared_mem", "launch__waves_per_multiprocessor",
]
TO_BYTES = {"byte": 1.0, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9, "Tbyte": 1e12}
TO_MS = {"ns": 1e-6, "us": 1e-3, "usecond": 1e-3, "ms": 1.0, "msecond": 1.0, "s": 1e3, "second": 1e3}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("report")
    ap.add_argument("out_prefix")
    ap.add_argument("--commit", default="?")
    ap.add_argument("--gpu", default="H100", help="card (and power limit) the report was captured on")
    ap.add_argument("--labels", nargs="*", default=[])
    ap.add_argument("--algorithmic", nargs="*", type=float, default=[], help="algorithmic bytes per launch, per kernel")
    args = ap.parse_args()
    raw = subprocess.run(["ncu", "-i", args.report, "--page", "raw", "--csv"], capture_output=True, text=True, check=True).stdout
    rows = list(csv.reader(io.StringIO(raw)))
    head, units, body = rows[0], rows[1], rows[2:]
    kernels = []
    for i, r in enumerate(body):
        rec = {"label": args.labels[i] if i < len(args.labels) else f"kernel {i}"}
        for name, unit, val in zip(head, units, r):
            short = name.split(".", 2)[-1] if name.count(".") >= 2 and name.split(".")[1].startswith("Triage") else name
            if name in ("Kernel Name", "Block Size", "Grid Size"):
                rec[name] = val
            elif short in KEEP or name in KEEP:
                key = short if short in KEEP else name
                try:
                    rec[key] = float(val.replace(",", ""))
                    rec[key + ".unit"] = unit
                except ValueError:
                    pass
        rd = rec.get("dram__bytes_read.sum", 0) * TO_BYTES.get(rec.get("dram__bytes_read.sum.unit", "byte"), 1)
        wr = rec.get("dram__bytes_write.sum", 0) * TO_BYTES.get(rec.get("dram__bytes_write.sum.unit", "byte"), 1)
        rec["traffic_bytes"] = rd + wr
        rec["time_ms"] = rec.get("gpu__time_duration.sum", 0) * TO_MS.get(rec.get("gpu__time_duration.sum.unit", "ms"), 1)
        if i < len(args.algorithmic):
            rec["algorithmic_bytes"] = args.algorithmic[i]
            rec["traffic_over_algorithmic"] = round(rec["traffic_bytes"] / args.algorithmic[i], 4)
        kernels.append(rec)
    doc = {"commit": args.commit, "command": f"ncu --set full --clock-control none --import-source on ... ({args.report})", "kernels": kernels}
    json.dump(doc, open(args.out_prefix + ".json", "w"), indent=1)
    with open(args.out_prefix + ".md", "w") as f:
        f.write(f"# ncu --set full, {args.gpu}, C2 state (16.06 GB, 1455 tensors), one launch each -- captured at commit {args.commit}\n\n")
        f.write("| kernel | time (ms) | DRAM read (GB) | DRAM write (GB) | traffic / algorithmic | DRAM % of ncu peak | regs | grid x block |\n|---|---|---|---|---|---|---|---|\n")
        for k in kernels:
            rd = k.get("dram__bytes_read.sum", 0) * TO_BYTES.get(k.get("dram__bytes_read.sum.unit", "byte"), 1) / 1e9
            wr = k.get("dram__bytes_write.sum", 0) * TO_BYTES.get(k.get("dram__bytes_write.sum.unit", "byte"), 1) / 1e9
            pct = k.get("gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", k.get("dram__throughput.avg.pct_of_peak_sustained_elapsed", 0))
            f.write(f"| {k['label']} `{k.get('Kernel Name', '')[:24]}` | {k['time_ms']:.3f} | {rd:.3f} | {wr:.3f} | {k.get('traffic_over_algorithmic', '')} | {pct:.1f} | "
                    f"{int(k.get('launch__registers_per_thread', 0))} | {k.get('Grid Size', '')} x {k.get('Block Size', '')} |\n")
        f.write("\nncu times are single cold launches under the profiler (not bench values); the bench number is CUDA-event timed in bench.py.\n")
    print(f"wrote {args.out_prefix}.json / .md with {len(kernels)} kernels")


if __name__ == "__main__":
    main()
