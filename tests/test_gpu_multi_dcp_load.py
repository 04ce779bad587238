"""Multi-GPU resharded torch.distributed.checkpoint load on the engine: Shard(0) DTensors saved on NCCL are loaded as
Shard(1) through ``CachedMetadataFileSystemReader(load_on_engine=True)``, bit-exact against the stock reader.
Needs >= 2 GPUs."""
import pytest
import torch

from _mp import run_ranks

pytestmark = [pytest.mark.gpu, pytest.mark.multigpu]


def _bits(t):
    t = t.detach().contiguous().cpu()
    return bytes(t.reshape(-1).view(torch.uint8).numpy())


def _w_dcp_reshard_load(rank, world, root):
    import torch.distributed.checkpoint as dcp
    from torch.distributed.device_mesh import init_device_mesh
    from torch.distributed.tensor import Shard, distribute_tensor

    from nvidia_resiliency_ext.checkpointing.async_ckpt.cached_metadata_filesystem_reader import CachedMetadataFileSystemReader

    mesh = init_device_mesh("cuda", (world,))
    g = torch.Generator(device="cuda").manual_seed(77)
    full = {"w": torch.randn(96 * world, 40 * world + 3, device="cuda", generator=g),
            "m": torch.randn(64 * world, 8 * world, device="cuda", generator=g).to(torch.bfloat16)}
    dcp.save({k: distribute_tensor(v, mesh, [Shard(0)]) for k, v in full.items()}, checkpoint_id=root)

    def targets():
        return {k: distribute_tensor(torch.zeros_like(v), mesh, [Shard(1)]) for k, v in full.items()}

    stock, eng = targets(), targets()
    dcp.load(stock, storage_reader=dcp.FileSystemReader(root))
    dcp.load(eng, storage_reader=CachedMetadataFileSystemReader(root, load_on_engine=True))
    torch.cuda.synchronize()
    for k, v in full.items():
        want = _bits(distribute_tensor(v, mesh, [Shard(1)]).to_local())
        assert _bits(stock[k].to_local()) == want and _bits(eng[k].to_local()) == want, k


def test_dcp_load_reshards_shard0_into_shard1(built_library, tmp_path):
    run_ranks(_w_dcp_reshard_load, min(torch.cuda.device_count(), 8), str(tmp_path / "ck"), backend="nccl")
