"""nvrx_xor_reduce on one GPU through the C ABI, bit-exact against numpy's XOR: source counts, sizes around vector and
grid boundaries, a range past 4 GiB, clearing of the sources, and the argument checks."""
import ctypes as C

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _lib():
    from nvidia_resiliency_ext.checkpointing.b200 import _cabi

    return _cabi.lib()


def _reduce(dst, srcs, nbytes, clear):
    arr = (C.c_void_p * max(len(srcs), 1))(*srcs)
    return _lib().nvrx_xor_reduce(dst, arr, len(srcs), nbytes, int(clear), torch.cuda.current_stream().cuda_stream)


def _random(nbytes, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randint(0, 256, (nbytes,), dtype=torch.uint8, device="cuda", generator=g)


@pytest.mark.parametrize("n", [1, 2, 3, 7])
@pytest.mark.parametrize("nbytes", [16, 4096 - 16, 4096, 4096 + 16, (3 << 20) + 4112, (17 << 20) - 48])
@pytest.mark.parametrize("clear", [False, True])
def test_xor_reduce_matches_numpy(built_library, n, nbytes, clear):
    srcs = [_random(nbytes, 10 * n + k) for k in range(n)]
    host = [s.cpu().numpy() for s in srcs]
    dst = torch.full((nbytes,), 0x5A, dtype=torch.uint8, device="cuda")
    assert _reduce(dst.data_ptr(), [s.data_ptr() for s in srcs], nbytes, clear) == 0
    torch.cuda.synchronize()
    want = host[0].copy()
    for h in host[1:]:
        want ^= h
    assert np.array_equal(dst.cpu().numpy(), want)
    for s, h in zip(srcs, host):
        assert np.array_equal(s.cpu().numpy(), np.zeros_like(h) if clear else h)


def test_xor_reduce_past_4gib(built_library):
    """Every byte of a range longer than 2^32: offsets that wrapped at 32 bits would XOR the head into the tail."""
    nbytes = (1 << 32) + (5 << 20) + 4096
    a = _random(nbytes, 1)
    b = _random(nbytes, 2)
    dst = torch.zeros(nbytes, dtype=torch.uint8, device="cuda")
    assert _reduce(dst.data_ptr(), [a.data_ptr(), b.data_ptr()], nbytes, False) == 0
    torch.cuda.synchronize()
    assert torch.equal(dst, torch.bitwise_xor(a, b))
    tail = slice((1 << 32) - 4096, nbytes)  # across the 2^32 boundary, checked on the host as well
    assert np.array_equal(dst[tail].cpu().numpy(), a[tail].cpu().numpy() ^ b[tail].cpu().numpy())
    assert _reduce(dst.data_ptr(), [a.data_ptr(), b.data_ptr()], nbytes, True) == 0
    torch.cuda.synchronize()
    assert int(a.count_nonzero()) == 0 and int(b.count_nonzero()) == 0
    del a, b, dst
    torch.cuda.empty_cache()


def test_xor_reduce_rejects_bad_arguments(built_library):
    from nvidia_resiliency_ext.checkpointing.b200._cabi import E_INVALID

    buf = torch.zeros(1 << 16, dtype=torch.uint8, device="cuda")
    base = buf.data_ptr()
    dst, s0, s1 = base, base + 16384, base + 32768
    before = buf.clone()
    assert _reduce(dst + 8, [s0, s1], 4096, False) == E_INVALID       # misaligned destination
    assert _reduce(dst, [s0 + 4, s1], 4096, False) == E_INVALID       # misaligned source
    assert _reduce(dst, [s0, s1], 4096 + 8, False) == E_INVALID       # bytes % 16 != 0
    assert _reduce(dst, [], 4096, False) == E_INVALID                 # n == 0
    assert _reduce(dst, [s0, dst + 4096 - 16], 4096, False) == E_INVALID  # dst overlaps a source (its last vector)
    assert _reduce(s0 + 4096 - 16, [s0], 4096, True) == E_INVALID       # ... or its first
    assert _reduce(dst, [s0, 0], 4096, False) == E_INVALID            # null source
    assert _reduce(dst, [s0] * 65, 4096, False) == E_INVALID          # more sources than one launch takes
    assert _reduce(dst, [s0, s1], 0, False) == 0                      # nothing to do, nothing launched
    torch.cuda.synchronize()
    assert torch.equal(buf, before)
