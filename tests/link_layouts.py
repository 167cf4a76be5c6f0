"""Test infrastructure: link-proof inputs built from their algebra instead of from two synthesised circuits.

A link proof shows that two wire polynomials a1, a2 agree on the link group D = {g^(offset + i) : i < size}, g the
generator of the 2^alignment-th roots of unity (1 <= size <= 2^alignment, so the roots are distinct; an offset of 2^alignment
or more names the roots of offset mod 2^alignment): q = (a1 - a2) / Z_D with Z_D = prod_{i < size} (X - g^(offset + i)).
`pair` draws the shorter polynomial at random and sets the longer one to it plus Z_D * q for a random q of len - size
coefficients, so that len1 and len2 take exactly the wanted values in either order.  `mismatch` adds c * Z_D / (X - root_j),
which vanishes on every root of the group but the j-th.

The device divides on the coset g' * H_N (N = 2^k >= len = max(len1, len2), at least 2) and reads an inexact division from
the quotient's coefficients [len - size, N); `CASES` are the layouts where that differs from the reference's `size`
successive synthetic divisions, each with the N, q_len and wrap it claims.  All values here are canonical Python integers
(`to_mont` gives the Montgomery limbs the ABI takes)."""
from __future__ import annotations

import random
from dataclasses import dataclass

import numpy as np

R = 0x30644E72E131A029B85045B68181585D2833E84879B97091_43E1F593F0000001
MONT = 1 << 256
MASK64 = (1 << 64) - 1


@dataclass(frozen=True)
class Case:
    name: str
    alignment: int
    offset: int
    size: int
    len1: int
    len2: int
    N: int       # the evaluation domain the device divides on
    q_len: int   # coefficients of the quotient
    identical: bool = False  # a1 = a2: zero quotient, identity commitments

    @property
    def len(self) -> int:
        return max(self.len1, self.len2)

    @property
    def wraps(self) -> bool:
        """the roots pass g^0 = 1 (still distinct: size <= 2^alignment)"""
        return self.offset % (1 << self.alignment) + self.size > 1 << self.alignment


CASES = [
    Case("size_one", 4, 3, 1, 10, 9, N=16, q_len=9),
    Case("q_len_one", 5, 2, 9, 10, 7, N=16, q_len=1),
    Case("whole_group", 4, 0, 16, 40, 33, N=64, q_len=24),              # Z_D = X^16 - 1
    Case("wraps", 3, 6, 5, 20, 12, N=32, q_len=15),                     # g^6, g^7, 1, g, g^2
    Case("wide_alignment", 12, 100, 7, 30, 20, N=32, q_len=23),         # 2^12-th roots, a 2^5 domain
    Case("no_slack", 6, 5, 10, 64, 50, N=64, q_len=54),                 # len = N
    Case("len1_lt_len2", 5, 20, 6, 21, 40, N=64, q_len=34),
    Case("len1_far_above_len2", 8, 40, 12, 1000, 17, N=1024, q_len=988),
    Case("len1_just_above_len2", 7, 100, 20, 129, 128, N=256, q_len=109),  # 129 = N/2 + 1: the most slack
    Case("identical", 5, 20, 6, 40, 40, N=64, q_len=34, identical=True),
    Case("largest_srs", 10, 1000, 3, (1 << 17) + 2, (1 << 17) - 7, N=1 << 18, q_len=(1 << 17) - 1),
    Case("offset_past_group", 5, (1 << 5) + 3, 6, 20, 14, N=32, q_len=14),    # the roots of offset 3
    Case("offset_2_63", 6, (1 << 63) + 5, 7, 24, 30, N=32, q_len=23),         # the roots of offset 5
    Case("whole_group_shifted", 3, 5, 8, 12, 9, N=16, q_len=4),               # Z_D = X^8 - 1, from g^5 round to g^4
    Case("alignment_zero", 0, 7, 1, 9, 6, N=16, q_len=8),                     # g = 1: the group {1}
    Case("alignment_28", 28, 12345, 4, 32, 25, N=32, q_len=28),               # 2^28-th roots, a 2^5 domain
]
BY_NAME = {c.name: c for c in CASES}


def domain_n(length: int) -> int:
    """N of `link` in plonk.cu: the smallest power of two >= length, at least 2"""
    n = 2
    while n < length:
        n *= 2
    return n


def generator(oracle, alignment: int) -> int:
    """g of the 2^alignment-th roots of unity, as the library and the oracle use it (`orc_domain_generator`)"""
    return oracle.limbs_to_int(oracle.domain_generator(alignment)) * pow(MONT, -1, R) % R


def roots(oracle, case: Case) -> list[int]:
    g = generator(oracle, case.alignment)
    r0 = pow(g, case.offset, R)
    return [r0 * pow(g, i, R) % R for i in range(case.size)]


def poly_mul(a: list[int], b: list[int]) -> list[int]:
    out = [0] * (len(a) + len(b) - 1)
    for i, x in enumerate(a):
        if x:
            for j, y in enumerate(b):
                out[i + j] = (out[i + j] + x * y) % R
    return out


def poly_add(a: list[int], b: list[int], sign: int = 1) -> list[int]:
    n = max(len(a), len(b))
    a, b = a + [0] * (n - len(a)), b + [0] * (n - len(b))
    return [(x + sign * y) % R for x, y in zip(a, b)]


def poly_eval(a: list[int], x: int) -> int:
    acc = 0
    for c in reversed(a):
        acc = (acc * x + c) % R
    return acc


def vanishing(rts: list[int]) -> list[int]:
    """coefficients of prod (X - root), lowest first"""
    z = [1]
    for r in rts:
        z = poly_mul(z, [(-r) % R, 1])
    return z


def div_linear(a: list[int], z: int) -> tuple[list[int], int]:
    """a = q (X - z) + rem: (q, rem)"""
    q = [0] * (len(a) - 1)
    run = 0
    for i in range(len(a) - 1, 0, -1):
        run = (run * z + a[i]) % R
        q[i - 1] = run
    return q, (run * z + a[0]) % R


def pair(oracle, case: Case, seed: int) -> tuple[list[int], list[int]]:
    """(a1, a2) of exactly len1 and len2 coefficients (non-zero top coefficients) with a1 - a2 = Z_D * q"""
    rng = random.Random(seed)
    short = min(case.len1, case.len2)
    base = [rng.randrange(R) for _ in range(short - 1)] + [rng.randrange(1, R)]
    if case.identical:
        assert case.len1 == case.len2
        return base, list(base)
    q = [rng.randrange(R) for _ in range(case.q_len - 1)] + [rng.randrange(1, R)]
    delta = poly_mul(vanishing(roots(oracle, case)), q)
    assert len(delta) == case.len
    a1, a2 = (poly_add(base, delta), base) if case.len1 >= case.len2 else (base, poly_add(base, delta, -1))
    assert (len(a1), len(a2)) == (case.len1, case.len2) and a1[-1] and a2[-1]
    return a1, a2


def mismatch(oracle, case: Case, a1: list[int], j: int, c: int) -> list[int]:
    """a1 + c * Z_D / (X - root_j): differs from a1 on root j of the group only"""
    rts = roots(oracle, case)
    other, rem = div_linear(vanishing(rts), rts[j])
    assert rem == 0 and len(other) <= len(a1)
    return poly_add(a1, [c * x % R for x in other])


def to_mont(vals: list[int]) -> np.ndarray:
    """(len, 4) uint64 Montgomery limbs"""
    out = np.zeros((len(vals), 4), dtype=np.uint64)
    raw = b"".join((v * MONT % R).to_bytes(32, "little") for v in vals)
    out[:] = np.frombuffer(raw, dtype=np.uint64).reshape(-1, 4)
    return out
