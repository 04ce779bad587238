"""ParityLocalCheckpointManager with parity_count = 2 on >= 3 GPUs (NCCL), one GPU per rank: the shared worker of
``test_gpu_multi_parity`` (saves over the fused P2P path and over NCCL, every save's parity bytes against the host
computation, m pack passes and one combine launch per save), with the first and the last member of the clique lost
together and rebuilt bit-exactly."""
import pytest
import torch

from _mp import run_ranks
from test_gpu_multi_parity import _w_parity

pytestmark = [pytest.mark.gpu, pytest.mark.multigpu,
              pytest.mark.skipif(torch.cuda.device_count() < 3, reason="needs >= 3 CUDA devices")]


@pytest.mark.parametrize("mode", ["p2p", "nccl"])
def test_rs_manager_save_and_rebuild_two_lost(built_library, shm_dir, mode):
    world = min(torch.cuda.device_count(), 8)
    run_ranks(_w_parity, world, str(shm_dir / mode), mode, 1, world, 2, [(0, world - 1)], backend="nccl")
