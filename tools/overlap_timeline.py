"""Timeline of one checkpoint inside a running training loop (nsys is not installed in this image): shows that the drain of
checkpoint N overlaps training steps N+1, N+2, ... instead of stalling them.

* training step = the dummy GEMM loop of bench.py (SURVEY 8d); every step is bracketed by CUDA events on the training stream;
* the drain is observed from the host: a thread samples the slot's progress word (advanced by the side stream after every
  256 MiB copy chunk) every ~0.2 ms;
* both clocks are tied together at one synchronisation point before the loop.

Prints a markdown table (one row per training step: start / end on the GPU, bytes in host memory at its end) and one JSON line.

    python tools/overlap_timeline.py > overlap_timeline.md
"""
import ctypes as C
import json
import os
import sys
import threading
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "nvidia-resiliency-ext_b200"))
import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

from bench import TrainingLoop, llama3_8b_shard_state  # noqa: E402


def main():
    torch.cuda.set_device(0)
    os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
    os.environ.setdefault("MASTER_PORT", "29588")
    dist.init_process_group("nccl", rank=0, world_size=1, device_id=torch.device("cuda", 0))
    from nvidia_resiliency_ext.checkpointing.async_ckpt.torch_ckpt import TorchAsyncCheckpoint

    dev = torch.device("cuda", 0)
    sd, total = llama3_8b_shard_state(dev)
    ckpt = TorchAsyncCheckpoint(persistent_queue=True)
    out = Path("/dev/shm") / f"nvrx_b200_tl_{os.getpid()}"
    out.mkdir(exist_ok=True)
    for i in range(2):  # warm: slots, plan, worker
        ckpt.async_save(sd, out / "w.pt")
        ckpt.finalize_async_save(blocking=True)
    loop = TrainingLoop(dev)
    steps_before, steps_after = 4, 14
    n = steps_before + steps_after
    marks = [torch.cuda.Event(enable_timing=True) for _ in range(n + 1)]
    samples, stop = [], threading.Event()
    state = {"ptr": None, "base": 0}

    def sampler():
        while not stop.is_set():
            if state["ptr"] is not None:
                samples.append((time.perf_counter(), C.c_uint64.from_address(state["ptr"]).value - state["base"]))
            time.sleep(0.0002)

    th = threading.Thread(target=sampler, daemon=True)
    th.start()
    torch.cuda.synchronize()
    t_sync = time.perf_counter()  # marks[0] completes "now" on the GPU: the two clocks meet here
    marks[0].record()
    t_call = t_ret = None
    for i in range(n):
        if i == steps_before:
            t_call = time.perf_counter()
            ckpt.async_save(sd, out / "ckpt.pt")
            t_ret = time.perf_counter()
            snap = next(iter(ckpt._pending.values()))
            state["base"] = snap.progress_target - snap.layout.total_bytes
            state["ptr"] = snap.slot.buf.progress_ptr
        loop.step(1)
        marks[i + 1].record()
    torch.cuda.synchronize()
    t_end = time.perf_counter()
    snap.wait()
    stop.set()
    th.join()
    ckpt.finalize_async_save(blocking=True)
    ckpt.close()
    import shutil

    shutil.rmtree(out, ignore_errors=True)

    ends = [marks[0].elapsed_time(marks[i + 1]) for i in range(n)]  # ms on the GPU clock since the sync point
    packed = snap.layout.total_bytes

    def drained_at(ms):
        t = t_sync + ms * 1e-3
        got = 0
        for ts, val in samples:
            if ts > t:
                break
            got = val
        return got

    first = next((ts for ts, v in samples if v > 0), None)
    last = next((ts for ts, v in samples if v >= packed), None)
    print(f"# One checkpoint inside a running training loop: the drain overlaps the following steps ({torch.cuda.get_device_name()}, C2 state, 16.06 GB)\n")
    print(f"training step = {loop.gemms} bf16 8192^3 GEMMs ({loop.step_ms:.1f} ms); `async_save` is called before step {steps_before}: "
          f"call took {(t_ret - t_call) * 1e3:.2f} ms on the host.\n")
    print("| step | GPU start (ms) | GPU end (ms) | duration (ms) | snapshot bytes in host memory at its end |")
    print("|---|---|---|---|---|")
    prev = 0.0
    for i, e in enumerate(ends):
        tag = " <- checkpoint taken at the start of this step (pack kernels run first in stream order)" if i == steps_before else ""
        print(f"| {i} | {prev:.1f} | {e:.1f} | {e - prev:.1f} | {drained_at(e) / 1e9:.2f} GB ({100 * drained_at(e) / packed:.0f} %){tag} |")
        prev = e
    base = sum(ends[i] - (ends[i - 1] if i else 0) for i in range(steps_before)) / steps_before
    ckpt_step = ends[steps_before] - ends[steps_before - 1]
    later = [ends[i] - ends[i - 1] for i in range(steps_before + 1, n)]
    summary = {
        "step_ms_before": round(base, 2), "step_ms_with_checkpoint": round(ckpt_step, 2),
        "extra_ms_in_checkpoint_step": round(ckpt_step - base, 2),
        "mean_step_ms_while_draining": round(sum(later[:8]) / len(later[:8]), 2),
        "drain_first_byte_ms_after_call": None if first is None else round((first - t_call) * 1e3, 2),
        "drain_complete_ms_after_call": None if last is None else round((last - t_call) * 1e3, 1),
        "steps_overlapped_by_the_drain": None if last is None else sum(1 for e in ends[steps_before:] if t_sync + e * 1e-3 < last),
        "drain_GBps": None if last is None or first is None else round(packed / (last - t_call) / 1e9, 1),
    }
    print("\n" + json.dumps(summary))
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
