"""Test infrastructure: edge operands of the BN254 fields and the values the library's field arithmetic must produce
for them, computed with Python integers.

Operands are Montgomery residues (canonical integers in [0, p)); the product of a and b is a * b * 2^-256 mod p.
`operands(p)` lists the values where multi-limb arithmetic goes wrong: 0, 1, 2, p - 1, p - 2, (p +- 1) / 2, R, R^2,
R^-1, p - R, every 2^k, 2^k - 1 and p - 2^k below 2^254, repeated 32-bit limb patterns, and for Fq random values in
[r, q) (which Fr-sized test vectors never reach).  `pairs(p)` combines them: the full cross product of a subset, every
value against a random partner in both orders, and pairs whose Montgomery product is exactly 1 or p - 1 (and the
field's one and minus one)."""
from __future__ import annotations

import random

import numpy as np

Q = 0x30644E72E131A029B85045B68181585D97816A916871CA8D3C208C16D87CFD47
R_FR = 0x30644E72E131A029B85045B68181585D2833E84879B97091_43E1F593F0000001
MONT = 1 << 256
MASK64 = (1 << 64) - 1

OP_MUL, OP_ADD, OP_SUB, OP_INV, OP_SQR, OP_MUL_ADD2, OP_MUL_SUB2 = range(7)


def operands(p: int) -> list[int]:
    R = MONT % p
    vals = [0, 1, 2, p - 1, p - 2, (p - 1) // 2, (p + 1) // 2, R, MONT * MONT % p, pow(MONT, -1, p), p - R]
    for k in range(254):
        vals += [1 << k, (1 << k) - 1, p - (1 << k)]
    for limb in (0xFFFFFFFF, 0xFFFFFFFE, 0x80000000, 0x7FFFFFFF, 0x00000001, 0xAAAAAAAA, 0x55555555, 0xDEADBEEF):
        vals.append(sum(limb << (32 * i) for i in range(8)) % p)
    if p == Q:
        rng = random.Random(0xF9)
        vals += [rng.randrange(R_FR, Q) for _ in range(64)]
    seen, out = set(), []
    for v in vals:
        assert 0 <= v < p
        if v not in seen:
            seen.add(v)
            out.append(v)
    return out


def pairs(p: int, cross: int = 96, seed: int = 0xE06E) -> tuple[list[int], list[int]]:
    """(a, b) operand lists of equal length; every entry is in [0, p)."""
    vals = operands(p)
    rng = random.Random(seed ^ p)
    sub = vals[:11] + rng.sample(vals[11:], cross - 11)
    a = [x for x in sub for _ in sub]
    b = [y for _ in sub for y in sub]
    for v in vals:
        r = rng.randrange(p)
        a += [v, r]
        b += [r, v]
    # Montgomery product exactly 1 or p - 1 (b = +-R / a), the largest and smallest results, and the field's one and
    # minus one (b = +-R^2 / a)
    R, R2 = MONT % p, MONT * MONT % p
    for v in [x for x in vals if x][:64] + [rng.randrange(1, p) for _ in range(64)]:
        inv = pow(v, -1, p)
        for t in (R, p - R, R2, p - R2):
            a.append(v)
            b.append(t * inv % p)
    return a, b


def expected(op: int, a: list[int], b: list[int], p: int) -> list[int]:
    """What field op `op` of b200_field_op returns (ops 5 / 6 pair element i with element n - 1 - i)."""
    ri = pow(MONT, -1, p)
    n = len(a)
    if op == OP_MUL:
        return [x * y * ri % p for x, y in zip(a, b)]
    if op == OP_ADD:
        return [(x + y) % p for x, y in zip(a, b)]
    if op == OP_SUB:
        return [(x - y) % p for x, y in zip(a, b)]
    if op == OP_INV:  # (x R^-1)^-1 R = x^-1 R^2; inv(0) = 0
        return [pow(x, -1, p) * MONT * MONT % p if x else 0 for x in a]
    if op == OP_SQR:
        return [x * x * ri % p for x in a]
    sign = 1 if op == OP_MUL_ADD2 else -1
    return [(a[i] * b[i] + sign * a[n - 1 - i] * b[n - 1 - i]) * ri % p for i in range(n)]


def to_array(vals) -> np.ndarray:
    out = np.zeros((len(vals), 4), dtype=np.uint64)
    for i, v in enumerate(vals):
        for k in range(4):
            out[i, k] = (v >> (64 * k)) & MASK64
    return out


def from_array(a: np.ndarray) -> list[int]:
    a = np.asarray(a, dtype=np.uint64).reshape(-1, 4)
    return [int(r[0]) | int(r[1]) << 64 | int(r[2]) << 128 | int(r[3]) << 192 for r in a]
