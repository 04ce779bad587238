"""The reference's OWN unit tests (tests/golden/ref_tests, verbatim copies) executed against this repo's mirror of the API:
``torchrun -m pytest`` with PYTHONPATH = nvidia-resiliency-ext_b200, one rank per GPU (SURVEY.md 7 step 2, VERDICT r1 item 5).

Reference files: tests/checkpointing/unit/test_async_save.py:26,58,123, test_basic_local.py:47,122, test_cleanup.py:46,
test_async_writer.py (the DCP writer, row f1)."""
import os
import subprocess
import sys
from pathlib import Path

import pytest
import torch

from conftest import PKG_ROOT, free_port

pytestmark = pytest.mark.gpu

FIXTURES = Path(__file__).resolve().parent / "golden" / "ref_tests"


def _kill_tagged(tag):
    """Processes THIS run started (they inherited its unique environment tag) that outlived it, e.g. a checkpoint worker of an
    aborted queue.  Exact pids, found by the tag, nothing else."""
    import signal

    for pid in [int(p) for p in os.listdir("/proc") if p.isdigit()]:
        try:
            env = open(f"/proc/{pid}/environ", "rb").read()
        except OSError:
            continue
        if f"NVRX_REFSUITE_TAG={tag}".encode() in env.split(b"\0") and pid != os.getpid():
            try:
                os.kill(pid, signal.SIGKILL)
            except OSError:
                pass


def run_reference_tests(files, world, extra=(), timeout=900, retries=0):
    """Run the given reference test files under torchrun against the mirror; returns pytest's stdout.  ``retries``: for groups
    that contain wall-clock assertions of the reference (test_cleanup.py asserts finalize_fn < 30 ms on a shared box).
    Output goes to files, not pipes: a process the tests leave behind would keep a pipe open and this call waiting for it."""
    for _ in range(retries):
        try:
            return run_reference_tests(files, world, extra, timeout, 0)
        except AssertionError:
            continue
    import tempfile
    import uuid

    tag = uuid.uuid4().hex
    env = dict(os.environ)
    env["PYTHONPATH"] = str(PKG_ROOT)  # the mirror, and nothing of this repo's own tests/ or oracle/
    env["NVRX_REFSUITE_TAG"] = tag
    env.pop("PYTEST_CURRENT_TEST", None)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}", "--master-addr", "127.0.0.1",
           "--master-port", str(free_port()), "-m", "pytest", "-q", "-x", "-p", "no:cacheprovider", "--confcutdir", str(FIXTURES),
           "--rootdir", str(FIXTURES), *[f"tests/checkpointing/unit/{f}" for f in files], *extra]
    with tempfile.TemporaryDirectory(prefix="nvrx_refsuite_") as tmp:
        out_path, err_path = Path(tmp) / "stdout", Path(tmp) / "stderr"
        code = None
        try:
            with open(out_path, "w") as so, open(err_path, "w") as se:
                code = subprocess.run(cmd, cwd=FIXTURES, env=env, stdin=subprocess.DEVNULL, stdout=so, stderr=se, timeout=timeout).returncode
        except subprocess.TimeoutExpired:
            pass
        finally:
            _kill_tagged(tag)
        stdout, stderr = out_path.read_text(errors="replace"), err_path.read_text(errors="replace")
    tail = stdout[-6000:] + "\n" + stderr[-3000:]
    assert code is not None, f"no result within {timeout} s\n{tail}"
    assert code == 0, tail
    return stdout


def passed_count(out):
    """N of pytest's closing ``N passed, ...`` line."""
    return int(out.rsplit(" passed", 1)[0].rsplit(None, 1)[-1])


def worlds():
    n = torch.cuda.device_count() if torch.cuda.is_available() else 0
    return [w for w in (1, 2) if w <= n]


def _needs(world):
    if world not in worlds():
        pytest.skip(f"needs >= {world} CUDA devices")


def _async_save_tests(world):
    out = run_reference_tests(["test_async_save.py"], world, timeout=240, retries=1)
    assert "3 passed" in out


def _local_checkpoint_tests(world):
    # test_find_latest_repl_disable asserts world_size >= 2 itself
    extra = ["-k", "not test_find_latest_repl_disable"] if world == 1 else []
    out = run_reference_tests(["test_basic_local.py", "test_cleanup.py"], world, extra, timeout=240, retries=1)
    assert " passed" in out and "failed" not in out


DCP_GROUPS = ["test_async_is_equivalent_to_sync", "test_invalid_async_setup", "test_errors_are_reported", "test_cached_metadata",
              "test_cached_data_structure", "test_cpu_shm_for_gpu_tensors", "test_async_cp_with_multiple_queue_and_abort"]


def _dcp_async_writer_tests(world):
    """All 13 cases of the reference's test_async_writer.py (the last -k pattern also selects ..._followed_by_delete).  Each
    group runs in a process of its own with its own time limit: in one process the file once did not finish within 900 s
    -- its last output came about 31 s in, then nothing.  Cause not found: every group passes on its own, and the same 13 scenarios replayed in ONE process on the stand-in device
    (queues with daemon / non-daemon workers, failing writers, caches, abort + resume) finish, so the host logic alone does
    not hang."""
    passed = 0
    for group in DCP_GROUPS:
        # a hang guard, not a speed check: the abort group takes about 145 s on a 16-core H100 host
        out = run_reference_tests(["test_async_writer.py"], world, ["-k", group], timeout=300, retries=1)
        assert " passed" in out and "failed" not in out, group
        passed += passed_count(out)
    assert passed == 13


# one rank first (what a 1-GPU box runs), the two-rank variants after them
def test_reference_async_save_tests():
    _async_save_tests(1)


def test_reference_local_checkpoint_tests():
    _local_checkpoint_tests(1)


def test_reference_dcp_async_writer_tests():
    _dcp_async_writer_tests(1)


def test_reference_local_checkpoint_tests_two_ranks():
    _needs(2)
    _local_checkpoint_tests(2)


def test_reference_async_save_tests_two_ranks():
    """Both ranks save the SAME path in this file (test_async_save.py:38): at two ranks it found the writer that truncated the
    file under the other rank's mapping (fixed: private name + rename); not repeated on GPUs since."""
    _needs(2)
    _async_save_tests(2)


def test_reference_dcp_async_writer_tests_two_ranks():
    _needs(2)
    _dcp_async_writer_tests(2)
