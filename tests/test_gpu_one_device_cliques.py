"""The erasure-coded and striped local checkpoint managers' device paths on ONE GPU: every rank of a clique is a process on
cuda:0 and the ranks talk over gloo.  The fused exchange still runs (the ranks import each other's exchange buffers through
CUDA IPC on the same device, the pack kernel stores into them), and so does the collective branch (pack, then
``all_to_all_single`` on device tensors).  Each run checks, with the shared workers of the multi-GPU tests, every save's
parity or fragment bytes against a host computation, the launches of the branch that ran, that the files hold the state
from before the live tensors were zeroed, the zero invariant of the exchange buffer after a smaller image, after a striped
save and with planted stale bytes, and a bit-exact rebuild of every lost set the code can recover (parity: every set of at
most m members of clique 0; striped: every single member).

What this does not show: NVLink timing and the stream-ordered NCCL barrier (gloo's CUDA all-reduce blocks the host, a
stronger barrier); ``test_gpu_multi*.py`` cover those on several GPUs."""
import pytest

from _mp import run_ranks
from test_gpu_multi import _w_sharded
from test_gpu_multi_parity import _w_parity

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("mode,F,m,jump,world", [
    ("p2p", 2, 1, 1, 2), ("p2p", 3, 1, 1, 3), ("p2p", 3, 2, 1, 3), ("p2p", 4, 2, 1, 4), ("p2p", 5, 3, 1, 5), ("p2p", 8, 2, 1, 8),
    ("p2p", 3, 2, 2, 6),  # two cliques, (0, 2, 4) and (1, 3, 5), on the one GPU
    ("nccl", 3, 2, 1, 3), ("nccl", 4, 1, 1, 4), ("nccl", 5, 3, 1, 5),
])
def test_parity_cliques_on_one_device(built_library, shm_dir, mode, F, m, jump, world):
    """``mode`` is ``NVRX_B200_EXCHANGE``: ``nccl`` takes the collective branch, which runs over gloo here."""
    run_ranks(_w_parity, world, str(shm_dir), mode, jump, F, m, None, backend="gloo", timeout=600)


@pytest.mark.parametrize("mode", ["p2p", "nccl"])
def test_striped_clique_on_one_device(built_library, shm_dir, mode):
    run_ranks(_w_sharded, 3, str(shm_dir), mode, 1, 3, [(0,), (1,), (2,)], backend="gloo", timeout=600)
