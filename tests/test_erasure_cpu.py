"""The erasure code of ParityLocalCheckpointManager (b200/erasure.py) on the host: field tables against an independent
shift-and-reduce multiply, the generator's MDS property, the stripe geometry at m = 1 against the striped manager's
mapping, and bit-exact recovery of every lost set the code claims to survive."""
import itertools
from types import SimpleNamespace

import numpy as np
import pytest

from nvidia_resiliency_ext.checkpointing.b200 import erasure as E


def slow_mul(a, b):
    r = 0
    for _ in range(8):
        if b & 1:
            r ^= a
        b >>= 1
        a <<= 1
        if a & 0x100:
            a ^= 0x11D
    return r


SLOW = np.array([[slow_mul(a, b) for b in range(256)] for a in range(256)], dtype=np.uint8)


def test_field_tables_match_shift_and_reduce():
    assert np.array_equal(E.MUL, SLOW)  # all 65,536 products
    assert E.mul(0x80, 2) == 0x1D and E.mul(2, 0x80) == 0x1D
    assert E.mul(0, 0x53) == 0 and E.mul(1, 0x53) == 0x53


def test_inverses():
    for a in range(1, 256):
        assert SLOW[a, E.inv(a)] == 1
    with pytest.raises(ZeroDivisionError):
        E.inv(0)
    rng = np.random.default_rng(1)
    for n in (1, 2, 3, 4):
        for _ in range(20):
            a = rng.integers(0, 256, (n, n), dtype=np.uint8)
            try:
                ai = E.mat_inv(a)
            except ValueError:
                assert det(a) == 0
                continue
            assert np.array_equal(E.matmul(a, ai), np.eye(n, dtype=np.uint8))


def det(a):
    """Determinant over GF(2^8) by elimination with the independent multiply (0 = singular)."""
    a = a.astype(np.int64).copy()
    n, d = a.shape[0], 1
    for c in range(n):
        piv = next((r for r in range(c, n) if a[r, c]), None)
        if piv is None:
            return 0
        a[[c, piv]] = a[[piv, c]]
        d = slow_mul(d, int(a[c, c]))
        pinv = next(x for x in range(1, 256) if slow_mul(int(a[c, c]), x) == 1)
        for r in range(c + 1, n):
            if a[r, c]:
                f = slow_mul(int(a[r, c]), pinv)
                a[r] ^= np.array([slow_mul(f, int(v)) for v in a[c]])
    return d


@pytest.mark.parametrize("F", range(2, 18))
def test_generator_is_mds(F):
    for m in range(1, min(F - 1, 4) + 1):
        k = F - m
        g = E.generator(m, k)
        assert g.shape == (m, k) and np.all(g[0] == 1)
        for t in range(1, min(m, k) + 1):
            for rows in itertools.combinations(range(m), t):
                for cols in itertools.combinations(range(k), t):
                    assert det(g[np.ix_(rows, cols)]) != 0, (F, m, rows, cols)


@pytest.mark.parametrize("F", range(2, 10))
def test_m1_geometry_is_the_xor_layout(F):
    from nvidia_resiliency_ext.checkpointing.local.ckpt_managers.sharded_local_manager import ShardedLocalCheckpointManager as S

    members = [3 * i + 1 for i in range(F)]
    striped = SimpleNamespace(_members=members)
    striped._others = lambda r: S._others(striped, r)
    code = E.StripeLayout(members, 1)
    for i, r in enumerate(members):
        assert code.held_stripes(r) == [i] and code.contributors(i) == striped._others(r)
        assert [code.holder(s, 0) for s in code.stripes_of(r)] == striped._others(r)
        for h in striped._others(r):
            assert code.slot(h, members.index(h), r) == S._slot_of_sender(striped, r, h)
        assert code.fragment_destinations(r, 0) == [(h, S._slot_of_sender(striped, r, h)) for h in striped._others(r)]


def encode(code, images, sb):
    """Parity rows of every holder, as a holder computes them from its exchange slots."""
    parity = {}
    for h in code.members:
        slots = [None] * (code.m * code.k)
        for i in code.members:
            for q, s in enumerate(code.stripes_of(i)):
                p = code.row_of(h, s)
                if p >= 0:
                    slots[code.slot(h, s, i)] = images[i][q * sb : (q + 1) * sb]
        assert all(x is not None for x in slots)
        parity[h] = np.concatenate(E.combine(code.encode_matrix(), slots))
    return parity


@pytest.mark.parametrize("F", range(2, 10))
def test_rebuild_plan_recovers_every_lost_set(F):
    rng = np.random.default_rng(F)
    members = list(range(10, 10 + F))
    for m in range(1, min(F - 1, 3) + 1):
        code = E.StripeLayout(members, m)
        sb = 48
        images = {r: rng.integers(0, 256, code.k * sb, dtype=np.uint8) for r in members}
        parity = encode(code, images, sb)
        for p in range(m):  # row 0 is the plain XOR of the stripe
            for h in members:
                s = code.held_stripes(h)[p]
                want = np.zeros(sb, dtype=np.uint8)
                for j, c in enumerate(code.contributors(s)):
                    q = code.stripes_of(c).index(s)
                    want ^= SLOW[code.G[p, j]][images[c][q * sb : (q + 1) * sb]]
                assert np.array_equal(parity[h][p * sb : (p + 1) * sb], want)
        for t in range(1, m + 1):
            for lost in itertools.combinations(members, t):
                steps = code.rebuild_plan(lost)
                got = {}
                for st in steps:
                    assert st.collector not in lost
                    srcs = []
                    for owner, kind, idx in st.sources:
                        assert owner not in lost
                        src = parity[owner] if kind == "parity" else images[owner]
                        srcs.append(src[idx * sb : (idx + 1) * sb])
                    assert len(srcs) == code.k and st.matrix.shape == (len(st.lost), code.k)
                    for (owner, q), out in zip(st.lost, E.combine(st.matrix, srcs)):
                        got[(owner, q)] = out
                assert sorted(got) == sorted((u, q) for u in lost for q in range(code.k))
                for (u, q), out in got.items():
                    assert np.array_equal(out, images[u][q * sb : (q + 1) * sb]), (F, m, lost, u, q)
        with pytest.raises(ValueError):
            code.rebuild_plan(members[: m + 1])
