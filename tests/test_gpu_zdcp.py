"""GPU test of the DCP async writer: the CUDA tensors of the plan go through ONE engine snapshot (pack kernel + drain), the
files must be byte-identical to a synchronous ``dcp.save`` and the trainer must be free to overwrite its tensors right after
scheduling (reference tests/checkpointing/unit/test_async_writer.py::test_async_is_equivalent_to_sync)."""
import filecmp
import os

import pytest
import torch
import torch.distributed.checkpoint as dcp
from torch.distributed.checkpoint import DefaultSavePlanner, FileSystemReader, FileSystemWriter

# (the writer's host side is covered by tests/test_dcp_async_cpu.py, byte for byte against the reference's own output)
pytestmark = pytest.mark.gpu  # part of the default suite


def _state(step=0):
    g = torch.Generator(device="cuda").manual_seed(5)
    return {
        "model": {f"w{i}": torch.randn(257 + i, 129, device="cuda", generator=g) + step for i in range(6)},
        "opt": {
            "m": torch.randn(1000, device="cuda", generator=g).to(torch.bfloat16),
            "ids": torch.arange(11, device="cuda", dtype=torch.int64),
            "host": torch.arange(5, dtype=torch.float32),  # stays on the host path
            "step": 3 + step,
        },
    }


@pytest.mark.parametrize("persistent", [True, False])
def test_dcp_async_on_engine_matches_sync(tmp_path, dist_1rank, persistent):
    from nvidia_resiliency_ext.checkpointing.async_ckpt.core import AsyncCallsQueue, AsyncRequest
    from nvidia_resiliency_ext.checkpointing.async_ckpt.filesystem_async import FileSystemWriterAsync
    from nvidia_resiliency_ext.checkpointing.async_ckpt.state_dict_saver import (
        save_state_dict_async_finalize,
        save_state_dict_async_plan,
    )

    q = AsyncCallsQueue(persistent=persistent)
    try:
        for step in range(2):
            state = _state(step)
            sync_dir, async_dir = tmp_path / f"sync{step}", tmp_path / f"async{step}"
            threads = 1 + step  # one thread is the case where stock PyTorch would pick its CUDA copy-ahead loader
            # (that loader orders the records of a file by size; per_thread_copy_ahead=0 selects the plan-order loader the
            # async writer uses, so that the files can be compared byte for byte)
            sync_writer = FileSystemWriter(sync_dir, thread_count=threads, per_thread_copy_ahead=0)
            dcp.save(state, storage_writer=sync_writer, planner=DefaultSavePlanner())
            writer = FileSystemWriterAsync(async_dir, thread_count=threads)
            ret = save_state_dict_async_plan(state, writer, None, 0, planner=DefaultSavePlanner())
            assert writer._snapshot is not None and len(writer._payload["cuda_indices"]) == 8
            save_fn, preload_fn, save_args = writer.get_save_function_and_args()
            q.schedule_async_request(
                AsyncRequest(save_fn, save_args, [lambda ret=ret: save_state_dict_async_finalize(*ret)], preload_fn=preload_fn)
            )
            for t in state["model"].values():  # training goes on
                t.fill_(-1.0)
            q.maybe_finalize_async_calls(blocking=True)
            assert writer._snapshot is None  # slot released by retrieve_write_results

            cmp = filecmp.dircmp(sync_dir, async_dir)
            assert not cmp.left_only and not cmp.right_only
            data = [f for f in cmp.common_files if f.endswith(".distcp")]
            _, mismatch, errors = filecmp.cmpfiles(sync_dir, async_dir, data, shallow=False)
            assert data and not mismatch and not errors, (mismatch, errors)

            expect = _state(step)
            got = {k: {kk: (torch.zeros_like(vv) if isinstance(vv, torch.Tensor) else None) for kk, vv in v.items()} for k, v in expect.items()}
            dcp.load(got, storage_reader=FileSystemReader(async_dir))
            for k, sub in expect.items():
                for kk, vv in sub.items():
                    if isinstance(vv, torch.Tensor):
                        assert torch.equal(got[k][kk], vv), (k, kk)
                    else:
                        assert got[k][kk] == vv
    finally:
        q.close()
