"""nvrx_gf_combine on one GPU through the C ABI, bit-exact against a numpy GF(2^8) oracle: coefficient matrices with 0, 1
and random entries, 1 to 64 sources into 1 to 4 destinations, sizes around the vector and grid boundaries, cleared
sources, an encode -> erase -> decode round trip on the device, a range past 4 GiB, and the argument checks."""
import ctypes as C

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _lib():
    from nvidia_resiliency_ext.checkpointing.b200 import _cabi

    return _cabi.lib()


def _combine(dsts, srcs, coef, nbytes, clear):
    coef = np.ascontiguousarray(np.asarray(coef, dtype=np.uint8)).reshape(-1)
    darr = (C.c_void_p * max(len(dsts), 1))(*dsts)
    sarr = (C.c_void_p * max(len(srcs), 1))(*srcs)
    carr = (C.c_uint8 * max(coef.size, 1)).from_buffer_copy(coef.tobytes() or b"\0")
    return _lib().nvrx_gf_combine(darr, len(dsts), sarr, len(srcs), carr, nbytes, int(clear), torch.cuda.current_stream().cuda_stream)


def _random(nbytes, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randint(0, 256, (nbytes,), dtype=torch.uint8, device="cuda", generator=g)


def _oracle(coef, host):
    """Shift-and-reduce tables, independent of the product's field code."""
    def mul(a, b):
        r = 0
        for _ in range(8):
            if b & 1:
                r ^= a
            b >>= 1
            a <<= 1
            if a & 0x100:
                a ^= 0x11D
        return r

    out = []
    for row in coef:
        acc = np.zeros_like(host[0])
        for c, h in zip(row, host):
            acc ^= np.array([mul(int(c), x) for x in range(256)], dtype=np.uint8)[h]
        out.append(acc)
    return out


def _coef(kind, nd, ns, seed):
    rng = np.random.default_rng(seed)
    if kind == "random":
        return rng.integers(0, 256, (nd, ns), dtype=np.uint8)
    if kind == "ones":
        return np.ones((nd, ns), dtype=np.uint8)
    c = rng.integers(0, 256, (nd, ns), dtype=np.uint8)  # mixed: zeros, ones and other values in every row
    c[:, ::3] = 0
    c[:, 1::3] = 1
    return c


@pytest.mark.parametrize("ns", [1, 2, 12, 64])
@pytest.mark.parametrize("nd", [1, 2, 3, 4])
@pytest.mark.parametrize("kind", ["random", "ones", "mixed"])
def test_gf_combine_matches_numpy(built_library, ns, nd, kind):
    nbytes = (1 << 16) + 4112
    coef = _coef(kind, nd, ns, 100 * ns + nd)
    srcs = [_random(nbytes, 7 * ns + s) for s in range(ns)]
    host = [s.cpu().numpy() for s in srcs]
    dsts = [torch.full((nbytes,), 0x5A, dtype=torch.uint8, device="cuda") for _ in range(nd)]
    assert _combine([d.data_ptr() for d in dsts], [s.data_ptr() for s in srcs], coef, nbytes, False) == 0
    torch.cuda.synchronize()
    for d, w in zip(dsts, _oracle(coef, host)):
        assert np.array_equal(d.cpu().numpy(), w)
    for s, h in zip(srcs, host):
        assert np.array_equal(s.cpu().numpy(), h)


@pytest.mark.parametrize("nbytes", [16, 4096 - 16, 4096, 4096 + 16, (3 << 20) + 4112, (17 << 20) - 48])
@pytest.mark.parametrize("clear", [False, True])
def test_gf_combine_sizes_and_clearing(built_library, nbytes, clear):
    ns, nd = 5, 3
    coef = _coef("mixed", nd, ns, nbytes % 1000)
    srcs = [_random(nbytes, 31 + s) for s in range(ns)]
    host = [s.cpu().numpy() for s in srcs]
    buf = torch.full((nd * nbytes + 64,), 0x5A, dtype=torch.uint8, device="cuda")  # destinations back to back, a guard after
    dsts = [buf.data_ptr() + d * nbytes for d in range(nd)]
    assert _combine(dsts, [s.data_ptr() for s in srcs], coef, nbytes, clear) == 0
    torch.cuda.synchronize()
    got = buf.cpu().numpy()
    for d, w in enumerate(_oracle(coef, host)):
        assert np.array_equal(got[d * nbytes : (d + 1) * nbytes], w)
    assert np.all(got[nd * nbytes :] == 0x5A)
    for s, h in zip(srcs, host):
        assert np.array_equal(s.cpu().numpy(), np.zeros_like(h) if clear else h)


def test_gf_combine_encode_erase_decode(built_library):
    """F = 8, m = 2: the parity of 6 data fragments, two of them erased and decoded from the parity and the other four."""
    from nvidia_resiliency_ext.checkpointing.b200 import erasure as E

    m, k, nbytes = 2, 6, (5 << 20) + 512
    g = E.generator(m, k)
    data = [_random(nbytes, 70 + j) for j in range(k)]
    want = [d.clone() for d in data]
    parity = torch.empty(m * nbytes, dtype=torch.uint8, device="cuda")
    assert _combine([parity.data_ptr() + p * nbytes for p in range(m)], [d.data_ptr() for d in data], g, nbytes, False) == 0
    lost, known = [1, 4], [0, 2, 3, 5]
    for j in lost:
        data[j].fill_(0xEE)
    a_inv = E.mat_inv(g[:, lost])
    dec = np.concatenate([a_inv, E.matmul(a_inv, g[:, known])], axis=1)
    srcs = [parity.data_ptr() + p * nbytes for p in range(m)] + [data[j].data_ptr() for j in known]
    assert _combine([data[j].data_ptr() for j in lost], srcs, dec, nbytes, False) == 0
    torch.cuda.synchronize()
    for j in range(k):
        assert torch.equal(data[j], want[j]), j


def test_gf_combine_past_4gib(built_library):
    """Every byte of a range longer than 2^32, compared on the device with a torch computation of the same combine."""
    from nvidia_resiliency_ext.checkpointing.b200 import erasure as E

    nbytes = (1 << 32) + (5 << 20) + 4096
    a = _random(nbytes, 1)
    b = _random(nbytes, 2)
    dst = torch.zeros(nbytes, dtype=torch.uint8, device="cuda")
    coef = [[1, 0x53]]
    assert _combine([dst.data_ptr()], [a.data_ptr(), b.data_ptr()], coef, nbytes, False) == 0
    mul53 = torch.from_numpy(E.MUL[0x53].copy()).cuda()
    step = 1 << 28
    for lo in range(0, nbytes, step):
        hi = min(nbytes, lo + step)
        assert torch.equal(dst[lo:hi], torch.bitwise_xor(a[lo:hi], mul53[b[lo:hi].long()])), lo
    tail = slice((1 << 32) - 4096, nbytes)  # across the 2^32 boundary, checked on the host as well
    assert np.array_equal(dst[tail].cpu().numpy(), _oracle(coef, [a[tail].cpu().numpy(), b[tail].cpu().numpy()])[0])
    assert _combine([dst.data_ptr()], [a.data_ptr(), b.data_ptr()], coef, nbytes, True) == 0
    torch.cuda.synchronize()
    assert int(a.count_nonzero()) == 0 and int(b.count_nonzero()) == 0
    del a, b, dst
    torch.cuda.empty_cache()


def test_gf_combine_rejects_bad_arguments(built_library):
    from nvidia_resiliency_ext.checkpointing.b200._cabi import E_INVALID

    buf = torch.zeros(1 << 17, dtype=torch.uint8, device="cuda")
    base = buf.data_ptr()
    d0, d1, s0, s1 = base, base + 16384, base + 32768, base + 49152
    before = buf.clone()
    c22 = [[1, 2], [3, 4]]
    assert _combine([d0 + 8, d1], [s0, s1], c22, 4096, False) == E_INVALID          # misaligned destination
    assert _combine([d0, d1], [s0 + 4, s1], c22, 4096, False) == E_INVALID          # misaligned source
    assert _combine([d0, d1], [s0, s1], c22, 4096 + 8, False) == E_INVALID          # bytes % 16 != 0
    assert _combine([d0, d1], [], [[], []], 4096, False) == E_INVALID               # n_src == 0
    assert _combine([], [s0, s1], [], 4096, False) == E_INVALID                     # n_dst == 0
    assert _combine([d0 + 512 * i for i in range(5)], [s0], [[1]] * 5, 512, False) == E_INVALID   # n_dst > 4
    assert _combine([d0], [s0] * 65, [[1] * 65], 4096, False) == E_INVALID          # n_src > 64
    assert _combine([d0, 0], [s0, s1], c22, 4096, False) == E_INVALID               # null destination
    assert _combine([d0, d1], [s0, 0], c22, 4096, False) == E_INVALID               # null source
    assert _combine([d0, d1], [s0, d1 + 4096 - 16], c22, 4096, True) == E_INVALID   # a destination overlaps a source
    assert _combine([d0, d0 + 4096 - 16], [s0, s1], c22, 4096, False) == E_INVALID  # destinations overlap
    darr = (C.c_void_p * 1)(d0)
    sarr = (C.c_void_p * 1)(s0)
    stream = torch.cuda.current_stream().cuda_stream
    assert _lib().nvrx_gf_combine(None, 1, sarr, 1, (C.c_uint8 * 1)(1), 4096, 0, stream) == E_INVALID   # null arrays
    assert _lib().nvrx_gf_combine(darr, 1, None, 1, (C.c_uint8 * 1)(1), 4096, 0, stream) == E_INVALID
    assert _lib().nvrx_gf_combine(darr, 1, sarr, 1, None, 4096, 0, stream) == E_INVALID
    assert _combine([d0, d1], [s0, s1], c22, 0, False) == 0                         # nothing to do, nothing launched
    torch.cuda.synchronize()
    assert torch.equal(buf, before)
