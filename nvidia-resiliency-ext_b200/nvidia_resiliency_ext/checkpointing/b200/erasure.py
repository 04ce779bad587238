"""The erasure code of ``ParityLocalCheckpointManager``: GF(2^8) arithmetic, the generator matrix and the stripe geometry.

Only this module decides the code and the layout; the manager asks it.

Field: GF(2^8) with the polynomial x^8+x^4+x^3+x^2+1 (0x11d), the field of ``nvrx_gf_combine``.

Code: a clique of F members keeps m parity fragments per stripe, k = F - m data fragments.  The generator ``G`` (m x k)
is a Cauchy matrix ``C[p][j] = 1 / (x_p ^ y_j)`` with ``x_p = p``, ``y_j = m + j``, every column scaled by ``1 / C[0][j]``
so that row 0 is all ones: row 0 is the XOR parity of the one-parity layout.  Scaling columns keeps every square
submatrix of a Cauchy matrix nonsingular, so the code is MDS: any m lost fragments of a stripe can be recovered.

Stripes: members ``c_0 .. c_{F-1}`` in clique order.  There are F stripes; parity row p of stripe s is held by
``c_{(s+p) mod F}`` (p < m); the contributors of stripe s are the other F - m members in clique order, contributor
position j uses column j of ``G``.  Member i cuts its packed image into k fragments; fragment q goes to the q-th stripe,
in clique order, that i contributes to.  At m = 1 this is the one-parity layout: stripe r is held by r and fragment q
goes to the q-th other member.
"""

from __future__ import annotations

from dataclasses import dataclass
from typing import Dict, List, Sequence, Tuple

import numpy as np

POLY = 0x11D


def _tables():
    exp = np.zeros(512, dtype=np.uint8)
    log = np.zeros(256, dtype=np.int32)
    x = 1
    for i in range(255):
        exp[i] = x
        log[x] = i
        x <<= 1
        if x & 0x100:
            x ^= POLY
    exp[255:510] = exp[:255]
    a = np.arange(256)
    mul = exp[(log[a][:, None] + log[a][None, :]) % 255]
    mul[0, :] = 0
    mul[:, 0] = 0
    return exp, log, mul.astype(np.uint8)


EXP, LOG, MUL = _tables()  # MUL[a, b] = a·b


def mul(a: int, b: int) -> int:
    return int(MUL[a, b])


def inv(a: int) -> int:
    if a == 0:
        raise ZeroDivisionError("0 has no inverse in GF(2^8)")
    return int(EXP[(255 - LOG[a]) % 255])


def matmul(a: np.ndarray, b: np.ndarray) -> np.ndarray:
    """Matrix product over GF(2^8) of uint8 matrices."""
    out = np.zeros((a.shape[0], b.shape[1]), dtype=np.uint8)
    for t in range(a.shape[1]):
        out ^= MUL[a[:, t][:, None], b[t, :][None, :]]
    return out


def mat_inv(a: np.ndarray) -> np.ndarray:
    """Inverse of a square uint8 matrix over GF(2^8) (Gauss-Jordan); raises ``ValueError`` if it is singular."""
    n = a.shape[0]
    w = np.concatenate([a.astype(np.uint8), np.eye(n, dtype=np.uint8)], axis=1)
    for col in range(n):
        piv = next((r for r in range(col, n) if w[r, col]), None)
        if piv is None:
            raise ValueError("singular matrix over GF(2^8)")
        w[[col, piv]] = w[[piv, col]]
        w[col] = MUL[inv(int(w[col, col])), w[col]]
        for r in range(n):
            if r != col and w[r, col]:
                w[r] ^= MUL[int(w[r, col]), w[col]]
    return w[:, n:].copy()


def combine(coef: np.ndarray, srcs: Sequence[np.ndarray]) -> List[np.ndarray]:
    """Host counterpart of ``nvrx_gf_combine``: ``out[d] = XOR over s of coef[d][s] · srcs[s]`` (uint8 arrays)."""
    coef = np.asarray(coef, dtype=np.uint8)
    out = [np.zeros_like(srcs[0]) for _ in range(coef.shape[0])]
    for s, src in enumerate(srcs):
        for d in range(coef.shape[0]):
            c = int(coef[d, s])
            if c == 1:
                out[d] ^= src
            elif c:
                out[d] ^= MUL[c][src]
    return out


def generator(m: int, k: int) -> np.ndarray:
    """The m x k generator matrix (see module docstring); row 0 is all ones."""
    if m < 1 or k < 1 or m + k > 256:
        raise ValueError(f"no generator for m={m}, k={k}")
    g = np.array([[inv(p ^ (m + j)) for j in range(k)] for p in range(m)], dtype=np.uint8)
    for j in range(k):
        g[:, j] = MUL[inv(int(g[0, j])), g[:, j]]
    return g


@dataclass(frozen=True)
class StripeRebuild:
    """How one stripe gets its lost fragments back.  ``sources`` are ``(member, kind, index)``: ``("parity", p)`` is parity
    row p as held by ``member``, ``("data", q)`` is fragment q of ``member``'s image; ``matrix`` (len(lost) x len(sources))
    maps them to the lost fragments, ``lost[i] = (owner, fragment index)``."""

    stripe: int
    collector: int
    sources: Tuple[Tuple[int, str, int], ...]
    lost: Tuple[Tuple[int, int], ...]
    matrix: np.ndarray


class StripeLayout:
    """The stripe geometry of one clique (``members`` in clique order) with ``m`` parity fragments per stripe."""

    def __init__(self, members: Sequence[int], m: int):
        self.members = list(members)
        self.F = len(self.members)
        if not 1 <= m < self.F:
            raise ValueError(f"parity_count must be between 1 and F-1 = {self.F - 1}, got {m}")
        self.m = m
        self.k = self.F - m
        self.G = generator(m, self.k)
        self._idx = {r: i for i, r in enumerate(self.members)}

    def holder(self, stripe: int, row: int) -> int:
        """Member that holds parity row ``row`` of ``stripe``."""
        return self.members[(stripe + row) % self.F]

    def row_of(self, holder: int, stripe: int) -> int:
        """Parity row of ``stripe`` that ``holder`` holds (``-1`` when it holds none)."""
        p = (self._idx[holder] - stripe) % self.F
        return p if p < self.m else -1

    def held_stripes(self, holder: int) -> List[int]:
        """Stripe of each parity row ``holder`` holds: entry p is the stripe of row p."""
        return [(self._idx[holder] - p) % self.F for p in range(self.m)]

    def contributors(self, stripe: int) -> List[int]:
        return [r for i, r in enumerate(self.members) if (i - stripe) % self.F >= self.m]

    def stripes_of(self, member: int) -> List[int]:
        """Stripe of each fragment of ``member``'s image: entry q is where fragment q goes."""
        i = self._idx[member]
        return [s for s in range(self.F) if (i - s) % self.F >= self.m]

    def column(self, member: int, stripe: int) -> int:
        return self.contributors(stripe).index(member)

    def slot(self, holder: int, stripe: int, sender: int) -> int:
        """Exchange slot at ``holder`` of ``sender``'s fragment of ``stripe``: ``p·k + j``."""
        return self.row_of(holder, stripe) * self.k + self.column(sender, stripe)

    def fragment_destinations(self, member: int, row: int) -> List[Tuple[int, int]]:
        """``(holder, slot)`` of every fragment q of ``member`` in pass ``row`` (to the row-``row`` holder of its stripe)."""
        out = []
        for s in self.stripes_of(member):
            h = self.holder(s, row)
            out.append((h, row * self.k + self.column(member, s)))
        return out

    def first_fragment(self, member: int) -> int:
        """Fragment a pack of ``member`` starts with: the one of stripe ``i+1``, so that at any moment the members of a
        clique store into different holders."""
        return self.stripes_of(member).index((self._idx[member] + 1) % self.F)

    def encode_matrix(self) -> np.ndarray:
        """Coefficients of the save combine at a holder: its ``m·k`` exchange slots into its m parity rows."""
        c = np.zeros((self.m, self.m * self.k), dtype=np.uint8)
        for p in range(self.m):
            c[p, p * self.k : (p + 1) * self.k] = self.G[p]
        return c

    def rebuild_plan(self, lost: Sequence[int]) -> List[StripeRebuild]:
        """Deterministic plan for a lost set of at most m members (see ``StripeRebuild``), stripes in increasing order."""
        lost_set = set(lost)
        if len(lost_set) > self.m:
            raise ValueError(f"{len(lost_set)} lost members, the code recovers at most {self.m}")
        plan = []
        for s in range(self.F):
            contrib = self.contributors(s)
            ucols = [j for j, r in enumerate(contrib) if r in lost_set]
            if not ucols:
                continue
            kcols = [j for j, r in enumerate(contrib) if r not in lost_set]
            rows = [p for p in range(self.m) if self.holder(s, p) not in lost_set][: len(ucols)]
            a_inv = mat_inv(self.G[np.ix_(rows, ucols)])
            b = self.G[np.ix_(rows, kcols)]
            matrix = np.concatenate([a_inv, matmul(a_inv, b)], axis=1) if kcols else a_inv
            sources = tuple((self.holder(s, p), "parity", p) for p in rows) + tuple(
                (contrib[j], "data", self.stripes_of(contrib[j]).index(s)) for j in kcols
            )
            owners = tuple((contrib[j], self.stripes_of(contrib[j]).index(s)) for j in ucols)
            plan.append(StripeRebuild(stripe=s, collector=self.holder(s, rows[0]), sources=sources, lost=owners, matrix=matrix))
        return plan

    def transfers(self, plan: Sequence[StripeRebuild]) -> Dict[Tuple[int, int], List[Tuple[int, int]]]:
        """``(sender, collector) -> [(step, source index), ...]``: the pieces of ``plan`` that travel, in plan order (a
        collector's own parity rows do not)."""
        out: Dict[Tuple[int, int], List[Tuple[int, int]]] = {}
        for t, step in enumerate(plan):
            for i, (owner, _, _) in enumerate(step.sources):
                if owner != step.collector:
                    out.setdefault((owner, step.collector), []).append((t, i))
        return out
