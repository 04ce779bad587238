"""Full replication (LocalCheckpointManager with CliqueReplicationStrategy) on ONE GPU: every rank of a clique is a process
on cuda:0 and the ranks talk over gloo.  The three branches of the packed exchange run -- ``p2p`` (the pack kernel stores
into every member's exchange buffer, imported through CUDA IPC on the same device, between two clique barriers), ``nccl``
(pack, then ``all_gather_into_tensor`` on device tensors, here over gloo) and ``stream`` (pack, then a chunked all-gather
through the two ring halves with a drain behind each chunk) -- and so does the retrieve of a lost member (packed
point-to-point message, one scatter).  The shared workers of ``test_gpu_multi`` compare everything bit for bit with host
copies of ``edge_state`` (an unaligned view, an odd-length bf16 tensor, an empty one, int64 and 0-d tensors, per-rank
sizes) taken before the save; the live tensors are zeroed on the training stream right after it.

What this does not show: NVLink timing, the stream-ordered NCCL barrier (gloo's CUDA collectives block the host, a
stronger barrier, so a missing device-side ordering before a collective goes unseen) and IPC across devices;
``test_gpu_multi.py`` covers those on several GPUs."""
import pytest

from _mp import run_ranks
from test_gpu_handoffs import cycles_per_ms  # noqa: F401  (fixture: the calibrated hold)
from test_gpu_multi import _w_allgather_batch, _w_replicated, _w_replicated_held

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("mode,F,small_chunks", [
    ("p2p", 2, False), ("p2p", 3, False), ("p2p", 8, False),
    ("nccl", 2, False), ("nccl", 3, False), ("nccl", 8, False),
    ("stream", 2, False), ("stream", 3, False), ("stream", 8, False),
    ("stream", 3, True),  # NVRX_B200_STREAM_CHUNK_MB=0: 512-byte chunks, many turns of the ring
])
def test_all_gather_batch_on_one_device(built_library, mode, F, small_chunks):
    run_ranks(_w_allgather_batch, F, mode, small_chunks, backend="gloo", timeout=600)


@pytest.mark.parametrize("mode", ["p2p", "nccl"])
@pytest.mark.parametrize("jump,F,world", [
    (1, 2, 2), (1, 3, 3), (1, 4, 4), (1, 8, 8),
    (2, 2, 4),  # two cliques, (0, 2) and (1, 3): group ranks differ from global ranks
])
def test_replicated_save_and_retrieve_on_one_device(built_library, shm_dir, mode, jump, F, world):
    """Kill sets: one member, then every member but the first (which then serves everyone)."""
    kills = [(F - 1,), tuple(range(1, F))] if F > 2 else [(1,)]
    run_ranks(_w_replicated, world, str(shm_dir), mode, jump, F, kills, backend="gloo", timeout=600)


@pytest.mark.parametrize("mode", ["p2p", "nccl"])
def test_replicated_structure_changes_on_one_device(built_library, shm_dir, mode):
    """A full state, a smaller one, then a larger one: the exchange buffer and the peer maps are regenerated; a fresh
    manager still finds and loads the last save, with no member lost and with one lost."""
    run_ranks(_w_replicated, 3, str(shm_dir), mode, 1, 3, [(), (0,)], True, backend="gloo", timeout=600)


@pytest.mark.parametrize("mode", ["p2p", "stream"])
def test_replicated_back_to_back_saves_with_held_drain(built_library, shm_dir, cycles_per_ms, mode):  # noqa: F811
    run_ranks(_w_replicated_held, 2, str(shm_dir), mode, cycles_per_ms, backend="gloo", timeout=600)


@pytest.mark.parametrize("F", [2, 3])
def test_replicated_zero_copy_on_one_device(built_library, shm_dir, F):
    """NVRX_B200_ZERO_COPY_REPLICAS=1: every member's slice lands in a slot of its own and is published by a hard link."""
    run_ranks(_w_replicated, F, str(shm_dir), "p2p", 1, F, [(F - 1,)], False, True, backend="gloo", timeout=600)
