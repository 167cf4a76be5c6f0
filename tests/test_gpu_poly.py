"""The stand-alone polynomial and vector primitives of plonk.cu (what the collaborative prover calls through the C ABI)
against Python integers: `b200_fr_poly_eval_device` (the chunked Horner scan of `eval_batch`, host-side path: the point
raised to CH per level on the host), `b200_fr_poly_div_linear_device` (`horner_suffix`, host-side path: the powers
z^1..z^CH filled on the host) and `b200_fr_vec_op`.

Lengths are chosen by the scan's level structure, with the chunk length CH read from plonk.cu: one chunk, chunk
boundaries, one element past them, up to 6 levels (2^20 + 1 coefficients; the prover's 2^17 + 3 need 5).  Points are 0,
1, r - 1, the multiplicative generator 5, roots of unity (a 16th root makes every level's point above the first 1) and
random points; coefficients random, all r - 1 (the largest residue), a single non-zero one at 0, 15, 16 and len - 1, or
all zero.  Every quotient coefficient and the value are checked."""
import ctypes as C
import os
import random
import re

import numpy as np
import pytest

import field_edges as fx

pytestmark = pytest.mark.gpu

R = fx.R_FR
MONT = fx.MONT
RINV = pow(MONT, -1, R)
ERR_INVALID = -1


def _chunk_length() -> int:
    with open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "renegade_b200", "csrc", "plonk.cu")) as f:
        m = re.search(r"constexpr int CH = (\d+);", f.read())
    assert m, "plonk.cu no longer defines CH"
    return int(m.group(1))


CH = _chunk_length()
# length -> levels of the chunked scan it is meant to reach
LEVELS = {1: 1, 2: 1, 3: 1, 15: 1, 16: 1, 17: 2, 31: 2, 32: 2, 33: 2, 255: 2, 256: 2, 257: 3, 4095: 3, 4096: 3, 4097: 4,
          65536: 4, 65537: 5, (1 << 20) + 1: 6}
LENGTHS = sorted(n for n in LEVELS if n <= 65537)


def levels(length: int) -> int:
    """kernel levels of `eval_batch` / `horner_suffix`: chunks of CH, then chunks of the chunk totals, ... down to one"""
    lv, n = 1, length
    while n > CH:
        n = (n + CH - 1) // CH
        lv += 1
    return lv


def test_lengths_reach_their_levels():
    assert CH == 16  # LEVELS is chosen for chunks of 16: a new CH needs new lengths
    for n, lv in LEVELS.items():
        assert levels(n) == lv, n
    # one element short of, exactly on, and one past every level's boundary
    for lv in range(1, 5):
        b = CH ** lv
        assert levels(b) == lv and levels(b + 1) == lv + 1
    assert {n % CH for n in (16, 32, 256, 4096, 65536)} == {0}


def points(ctx) -> dict:
    """canonical evaluation points"""
    out = {"0": 0, "1": 1, "r-1": R - 1, "5": 5}
    for k in (4, 8, 12, 20, 28):
        w = fx.from_array(ctx.domain_generator(k))[0] * RINV % R
        assert pow(w, 1 << k, R) == 1 and pow(w, 1 << (k - 1), R) == R - 1
        out[f"w{k}"] = w
    rng = random.Random(0x90117)
    out["rand0"], out["rand1"] = rng.randrange(R), rng.randrange(R)
    return out


def patterns(n: int) -> dict:
    """stored (Montgomery) coefficient residues"""
    rng = random.Random(0xC0EF + n)
    out = {"random": [rng.randrange(R) for _ in range(n)], "max": [R - 1] * n, "zero": [0] * n}
    for i in sorted({0, 15, 16, n - 1}):
        if i < n:
            v = [0] * n
            v[i] = rng.randrange(1, R)
            out[f"one_at_{i}"] = v
    return out


def to_device(stored: list[int]):
    import torch
    raw = b"".join(v.to_bytes(32, "little") for v in stored)
    return torch.frombuffer(bytearray(raw), dtype=torch.int64).reshape(-1, 4).cuda()


def limbs(v: int) -> np.ndarray:
    return fx.to_array([v])[0].copy()


def eval_device(ctx, d, n: int, z_stored: int) -> int:
    import torch
    from renegade_b200 import _lib
    out = np.full(4, 0xFFFFFFFFFFFFFFFF, dtype=np.uint64)
    zz = limbs(z_stored)
    torch.cuda.synchronize()
    _lib.check(ctx._lib.b200_fr_poly_eval_device(ctx._h, C.c_void_p(d.data_ptr() if n else 0), n, zz.ctypes.data_as(C.c_void_p),
                                                  out.ctypes.data_as(C.c_void_p)))
    return fx.from_array(out)[0]


def div_device(ctx, d, n: int, z_stored: int) -> bytes:
    import torch
    from renegade_b200 import _lib
    q = torch.full((n - 1 + 8, 4), -1, dtype=torch.int64, device="cuda")  # 8 guard rows after the quotient
    zz = limbs(z_stored)
    torch.cuda.synchronize()
    _lib.check(ctx._lib.b200_fr_poly_div_linear_device(ctx._h, C.c_void_p(d.data_ptr()), n, zz.ctypes.data_as(C.c_void_p),
                                                        C.c_void_p(q.data_ptr())))
    host = q.cpu().numpy().view(np.uint64)
    assert (host[n - 1:] == np.uint64(0xFFFFFFFFFFFFFFFF)).all(), "wrote past the quotient"
    return host[:n - 1].tobytes()


def suffix(coeffs: list[int], z: int) -> list[int]:
    """S[j] = sum_{i >= j} p_i z^(i - j), canonical: S[0] = p(z), S[1:] = the quotient of p / (X - z)"""
    s = [0] * len(coeffs)
    run = 0
    for i in range(len(coeffs) - 1, -1, -1):
        run = (run * z + coeffs[i]) % R
        s[i] = run
    return s


def stored_bytes(canon: list[int]) -> bytes:
    return b"".join((v * MONT % R).to_bytes(32, "little") for v in canon)


def check_one(ctx, d, stored, canon, z, label):
    n = len(stored)
    s = suffix(canon, z)
    zs = z * MONT % R
    assert eval_device(ctx, d, n, zs) == s[0] * MONT % R, ("value", label)
    if n >= 2:
        got = div_device(ctx, d, n, zs)
        want = stored_bytes(s[1:])
        if got != want:
            bad = [j for j in range(n - 1) if got[32 * j:32 * j + 32] != want[32 * j:32 * j + 32]]
            raise AssertionError(("quotient", label, len(bad), bad[:8]))


@pytest.mark.parametrize("n", LENGTHS)
def test_eval_and_div_linear_match_horner(ctx, n):
    assert levels(n) == LEVELS[n]
    pts = points(ctx)
    pats = patterns(n)
    if n <= 4097:  # every point with every pattern
        combos = [(p, z) for p in pats for z in pts]
    else:  # every point on random coefficients, every pattern at a random point and at the 16th root of unity
        combos = [("random", z) for z in pts] + [(p, z) for p in pats if p != "random" for z in ("rand0", "w4")]
    for pname in dict.fromkeys(p for p, _ in combos):
        stored = pats[pname]
        canon = [v * RINV % R for v in stored]
        d = to_device(stored)
        for z in (z for p, z in combos if p == pname):
            check_one(ctx, d, stored, canon, pts[z], (n, pname, z))


def test_six_levels(ctx):
    """2^20 + 1 coefficients: every quotient coefficient (the chunk boundaries of all six levels among them), the value,
    and p(x) = q(x)(x - z) + p(z) at random x from the device quotient"""
    n = (1 << 20) + 1
    assert levels(n) == 6
    rng = random.Random(0x6)
    canon = [rng.randrange(R) for _ in range(n)]
    stored = [v * MONT % R for v in canon]
    d = to_device(stored)
    z = rng.randrange(R)
    s = suffix(canon, z)
    assert eval_device(ctx, d, n, z * MONT % R) == s[0] * MONT % R
    got = div_device(ctx, d, n, z * MONT % R)
    arr = np.frombuffer(got, dtype=np.uint64).reshape(-1, 4)
    q = [(int(r[0]) | int(r[1]) << 64 | int(r[2]) << 128 | int(r[3]) << 192) * RINV % R for r in arr]
    for j in sorted({0, 1, n - 2} | {b + e for b in (CH, CH ** 2, CH ** 3, CH ** 4, CH ** 5) for e in (-2, -1, 0) if b + e < n - 1}):
        assert q[j] == s[j + 1], j
    assert q == s[1:]
    for _ in range(2):
        x = rng.randrange(R)
        assert suffix(canon, x)[0] == (suffix(q, x)[0] * (x - z) + s[0]) % R


def test_error_paths(ctx):
    import torch
    d = to_device([1, 2, 3])
    assert eval_device(ctx, None, 0, 5) == 0  # the empty polynomial is 0
    zz = limbs(5)
    q = torch.zeros((4, 4), dtype=torch.int64, device="cuda")
    for n in (0, 1):
        rc = ctx._lib.b200_fr_poly_div_linear_device(ctx._h, C.c_void_p(d.data_ptr()), n, zz.ctypes.data_as(C.c_void_p),
                                                     C.c_void_p(q.data_ptr()))
        assert rc == ERR_INVALID, n
    assert not q.any()


VEC_OPS = {0: fx.OP_ADD, 1: fx.OP_SUB, 2: fx.OP_MUL}  # b200_fr_vec_op's op -> field_edges op


def vec_op(ctx, op: int, a, b, scalar: bool, n: int):
    import torch
    from renegade_b200 import _lib
    out = torch.full((n + 64, 4), -1, dtype=torch.int64, device="cuda")  # 64 guard rows
    torch.cuda.synchronize()
    _lib.check(ctx._lib.b200_fr_vec_op(ctx._h, op, C.c_void_p(a.data_ptr()), C.c_void_p(b.data_ptr()), int(scalar), n,
                                       C.c_void_p(out.data_ptr())))
    host = out.cpu().numpy().view(np.uint64)
    assert (host[n:] == np.uint64(0xFFFFFFFFFFFFFFFF)).all(), "wrote past n"
    return fx.from_array(host[:n])


@pytest.mark.parametrize("n", [1, 255, 256, 257, None], ids=["1", "255", "256", "257", "all"])
def test_vec_op_on_edge_operands(ctx, n):
    """add, sub and Montgomery product, with a vector and with a scalar b, on the edge operands of field_edges.py"""
    a, b = fx.pairs(R)
    if n is not None:
        a, b = a[:n], b[:n]
    n = len(a)
    da, db = to_device(a), to_device(b)
    rng = random.Random(0x7EC)
    scalars = [0, 1, 2, R - 1, R - 2, MONT % R, R - MONT % R, MONT * MONT % R, rng.randrange(R)]
    for op, fop in VEC_OPS.items():
        got = vec_op(ctx, op, da, db, False, n)
        assert got == fx.expected(fop, a, b, R), (op, "vector")
        for s in scalars:
            got = vec_op(ctx, op, da, to_device([s]), True, n)
            assert got == fx.expected(fop, a, [s] * n, R), (op, hex(s))
