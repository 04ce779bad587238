"""GPU CRC-32 (csrc/crc_kernels.cuh) on the device.  The arithmetic, the tables and the CPU-only chaining are covered without a
GPU (tests/test_crc_cpu.py runs the kernel's own device functions lane by lane on the host); what is left for the GPU is the
kernel's indexing / launch and the engine plumbing."""
import ctypes as C
import os
import zipfile
import zlib

import numpy as np
import pytest
import torch

from oracle import crc_oracle as co

pytestmark = pytest.mark.gpu  # part of the default suite


def test_kernel_values_match_zlib(built_library, monkeypatch):
    monkeypatch.delenv("NVRX_B200_CRC_VARIANT", raising=False)  # crc_chunks_private<32>, the default kernel
    _check_kernel_values_match_zlib()


def test_shared_kernel_values_match_zlib(built_library, monkeypatch):
    monkeypatch.setenv("NVRX_B200_CRC_VARIANT", "shared")  # crc_chunks<8>: one copy of the tables per CTA, read at every launch
    _check_kernel_values_match_zlib()


def _check_kernel_values_match_zlib():
    from nvidia_resiliency_ext.checkpointing.b200.engine import CrcPlan, finish_crcs

    g = torch.Generator(device="cuda").manual_seed(9)
    sizes = [0, 4, 511, 512, 513, 65536, 65536 + 512, 5 * 65536 + 3 * 512 + 77, 1 << 24, 700, (1 << 26) + 12345]
    offsets, cur = [], 0
    for i, nb in enumerate(sizes):
        cur = -(-cur // 512) * 512 + (8 if i == 9 else 0)
        offsets.append(cur)
        cur += nb
    buf = torch.randint(0, 256, (cur + 64,), dtype=torch.uint8, device="cuda", generator=g)
    host = buf.cpu().numpy()
    plan = CrcPlan(offsets, sizes, torch.cuda.current_device())
    chunks = co.chunks_of(offsets, sizes)
    assert plan.n_values == len(chunks)
    values = torch.zeros(plan.n_values + 2, dtype=torch.int32).pin_memory()
    ready = torch.zeros(1, dtype=torch.int64).pin_memory()
    stream = torch.cuda.current_stream().cuda_stream
    for rep in (1, 2):  # the second run reuses the uploaded chunk list
        plan.run(buf.data_ptr(), values.data_ptr(), ready.data_ptr(), 1000 + rep, stream)
        torch.cuda.synchronize()
        assert int(ready[0]) == 1000 + rep
        got = values[: plan.n_values].numpy().view(np.uint32)
        step = max(1, len(chunks) // 300)
        for k in list(range(0, len(chunks), step)) + [len(chunks) - 1]:
            off, rows, _ = chunks[k]
            assert int(got[k]) == co.chunk_value(host[off : off + rows * 512].tobytes()), (k, off, rows)
        crcs = finish_crcs(offsets, sizes, values.data_ptr(), plan.n_values, host.ctypes.data)
        assert crcs == [zlib.crc32(host[o : o + n].tobytes()) for o, n in zip(offsets, sizes)]
    plan.close()


@pytest.mark.parametrize("zero_copy", ["1", "0"])
def test_published_checkpoint_has_valid_record_checksums(shm_dir, dist_1rank, built_library, monkeypatch, zero_copy):
    from nvidia_resiliency_ext.checkpointing.async_ckpt.torch_ckpt import TorchAsyncCheckpoint

    monkeypatch.setenv("NVRX_B200_ZERO_COPY", zero_copy)
    monkeypatch.setenv("NVRX_B200_GPU_CRC", "1")
    monkeypatch.setenv("NVRX_B200_ZIP_CRC", "0")
    g = torch.Generator(device="cuda").manual_seed(2)
    sd = {f"p{i}": torch.randn(1000 + i, 129, device="cuda", generator=g) for i in range(20)}
    sd["step"] = torch.tensor(7.0, device="cuda")
    ckpt = TorchAsyncCheckpoint(persistent_queue=True)
    try:
        for it in range(2):
            path = shm_dir / f"crc{it}.pt"
            ckpt.async_save(sd, path)
            ckpt.finalize_async_save(blocking=True)
            assert os.stat(path).st_nlink == (2 if zero_copy == "1" else 1)  # hard link to the slot, or a copied container
            archive = "archive" if zero_copy == "1" else f"crc{it}"
            with zipfile.ZipFile(path) as zf:
                for n in zf.namelist():
                    if not n.endswith("/.pad"):
                        zf.read(n)  # raises on a wrong CRC
                assert zf.getinfo(f"{archive}/data/0").CRC == zlib.crc32(sd["p0"].cpu().numpy().tobytes())
            loaded = torch.load(path, weights_only=False)
            assert all(torch.equal(loaded[k], v.cpu()) for k, v in sd.items())
            sd["p0"].add_(1.0)
    finally:
        ckpt.close()


def test_restore_verification_catches_a_flipped_bit(tmp_path, dist_1rank, built_library, monkeypatch):
    """NVRX_B200_VERIFY_RESTORE=1: the checksum kernel sums what arrived in HBM and compares with the file's directory."""
    from nvidia_resiliency_ext.checkpointing.b200._cabi import SnapError
    from nvidia_resiliency_ext.checkpointing.local.basic_state_dict import BasicTensorAwareStateDict
    from nvidia_resiliency_ext.checkpointing.local.ckpt_managers.local_manager import LocalCheckpointManager

    monkeypatch.setenv("NVRX_B200_VERIFY_RESTORE", "1")
    monkeypatch.setenv("NVRX_B200_ZIP_CRC", "1")  # the copying writer fills the CRC fields in (CPU threads)
    g = torch.Generator(device="cuda").manual_seed(4)
    sd = {f"p{i}": torch.randn(513 + i, 255, device="cuda", generator=g) for i in range(8)}
    mgr = LocalCheckpointManager(tmp_path)
    mgr.save(BasicTensorAwareStateDict({k: v.clone() for k, v in sd.items()}), 3, is_async=False)
    assert mgr.find_latest() == 3
    loaded, _ = mgr.load()  # intact file: passes
    assert all(torch.equal(loaded.state_dict[k], v) for k, v in sd.items())
    path = mgr._local_ckpt_path_from_id(mgr._ckpt_id(3))
    reader = torch._C.PyTorchFileReader(str(path))
    off = reader.get_record_offset("data/5") + 70_001
    del reader
    with open(path, "r+b") as fh:
        fh.seek(off)
        byte = fh.read(1)
        fh.seek(off)
        fh.write(bytes([byte[0] ^ 0x10]))
    mgr2 = LocalCheckpointManager(tmp_path)
    assert mgr2.find_latest() == 3
    with pytest.raises(SnapError, match="crc32 mismatch"):
        mgr2.load()
