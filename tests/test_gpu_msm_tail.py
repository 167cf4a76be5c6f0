"""GPU: the bucket reduction of throughput plans — the serial tree level reading the segment sums, msm_tail_kernel
(row / column sums as warp-local sums) and msm_tail_bits_kernel (the c - 1 bit sums per window) — at the windows and batch
sizes the prover runs, against the oracle or the known-discrete-log closed form.

At c = 15 the rows of a window have L = 128 buckets, at c = 16 and 17 L = 256; the serial level adds 8 neighbouring
buckets (rows) or rows (columns), the tail sums the L / 8 partials of a row and the partials of a column, lanes of one
warp meeting in shuffle levels.  The shapes: random vectors in batches of 1, 5 and 64 with identity members, n = 8 L + 1
points; every bucket empty; every bucket holding the same point (the doubling path at every level); a row and a column
whose two serial partials are P and -P (the identity from a cancellation inside the tail); a bucket cut into more
segments than the sequential combine takes (its sum comes from msm_heavy_combine_kernel)."""
import ctypes as C
import random

import numpy as np
import pytest

import msm_digits as md
import renegade_b200 as rb

pytestmark = pytest.mark.gpu

R = md.R
Q = 0x30644E72E131A029B85045B68181585D97816A916871CA8D3C208C16D87CFD47
SEED = 0x7A11
WINDOWS = [15, 16, 17]


def row_len(c: int) -> int:
    return 1 << (c // 2)  # L = 2^ceil((c - 1) / 2)


def msm_batch(ctx, bases, vectors: np.ndarray, stride: int):
    """b200_msm_batch_device over `vectors` (batch, n, 4) canonical scalars laid out `stride` apart on the device."""
    import torch
    from renegade_b200 import _lib
    batch, n = vectors.shape[0], vectors.shape[1]
    s = np.zeros((batch, stride, 4), dtype=np.uint64)
    s[:, :n] = vectors
    t = torch.from_numpy(s.view(np.int64)).cuda()
    torch.cuda.synchronize()
    out = np.zeros((batch, 8), dtype=np.uint64)
    inf = (C.c_int * batch)()
    _lib.check(ctx._lib.b200_msm_batch_device(ctx._h, bases._h, 0, C.c_void_p(t.data_ptr()), n, stride, batch, 0,
                                              out.ctypes.data_as(C.c_void_p), inf))
    return out, [bool(v) for v in inf]


def generator(pyoracle) -> np.ndarray:
    return np.frombuffer(pyoracle.encode_g1_mont(pyoracle.G1_GEN), dtype=np.uint64).copy()


def negate(pts: np.ndarray) -> np.ndarray:
    out = pts.copy()
    for i in range(out.shape[0]):
        y = sum(int(out[i, 4 + k]) << (64 * k) for k in range(4))
        out[i, 4:] = [((Q - y) >> (64 * k)) & ((1 << 64) - 1) for k in range(4)]
    return out


@pytest.mark.parametrize("batch", [1, 5, 64])
@pytest.mark.parametrize("c", WINDOWS)
def test_random_batches(ctx, oracle, c, batch):
    n = 8 * row_len(c) + 1  # any n: the reduction's groups are over the 2^(c-1) buckets of a window, all full whatever n is
    pts = oracle.known_dlog_bases(SEED, n)
    bases = ctx.load_bases(pts, window_bits=c)
    assert bases.plan == {"window_bits": c, "digits": md.num_windows(c), "physical_windows": 1, "tables": md.num_windows(c)}
    vectors = np.stack([oracle.splitmix_fr(0x7A1 + 97 * c + i, n, False) for i in range(batch)])
    if batch > 1:
        vectors[1] = 0
        vectors[-1] = 0
    out, inf = msm_batch(ctx, bases, vectors, n + 3)
    for b in range(batch):
        exp, einf = oracle.msm(pts, vectors[b])
        assert einf == (batch > 1 and b in (1, batch - 1))
        assert inf[b] == einf and (out[b] == exp).all(), b


@pytest.mark.parametrize("c", WINDOWS)
def test_every_bucket_empty(ctx, oracle, c):
    n = 8 * row_len(c) + 1
    bases = ctx.load_bases(oracle.known_dlog_bases(SEED, n), window_bits=c)
    out, inf = msm_batch(ctx, bases, np.zeros((5, n, 4), dtype=np.uint64), n)
    assert all(inf) and not out.any()


@pytest.mark.parametrize("c", WINDOWS)
def test_every_bucket_equal(ctx, oracle, pyoracle, c):
    """Every base is G and scalar i is i + 1 < 2^(c-1): each of the window's 2^(c-1) buckets holds exactly G and the
    other windows are empty, so every addition of the reduction adds two equal points."""
    half = 1 << (c - 1)
    g = generator(pyoracle)
    pts = np.tile(g, (half, 1))
    s = oracle.ints_to_array(range(1, half + 1))
    counts = md.bucket_counts_np(s, c)
    assert (counts[:half] == 1).all() and counts.sum() == half
    bases = ctx.load_bases(pts, window_bits=c)
    exp, einf = oracle.g1_mul(g, False, oracle.int_to_limbs(half * (half + 1) // 2 % R))
    assert not einf
    out, inf = ctx.msm(bases, s)
    assert not inf and (out == exp).all()
    out, inf = msm_batch(ctx, bases, np.stack([s, np.zeros_like(s), s]), half)
    assert inf == [False, True, False] and (out[0] == exp).all() and (out[2] == exp).all()


@pytest.mark.parametrize("c", WINDOWS)
def test_opposite_partials_cancel(ctx, oracle, c):
    """P in bucket 1 (row 0, column 1) and -P in bucket 9 (row 0, column 9) make row 0's first two serial partials P and
    -P; Q in bucket L (row 1, column 0) and -Q in bucket 9 L (row 9, column 0) make column 0's first two partials Q and -Q.
    Nothing else is in row 0 or column 0, so both sums are the identity, reached by a cancellation inside the tail."""
    L = row_len(c)
    p = oracle.known_dlog_bases(SEED, 2)
    pts = np.concatenate([p[:1], negate(p[:1]), p[1:], negate(p[1:])])
    s = oracle.ints_to_array([2, 10, L + 1, 9 * L + 1])  # digit d lands in bucket d - 1
    counts = md.bucket_counts_np(s, c)
    assert [int(counts[b]) for b in (1, 9, L, 9 * L)] == [1, 1, 1, 1] and counts.sum() == 4
    assert counts[:L].sum() == 2 and counts[::L].sum() == 2  # row 0 holds P and -P only, column 0 Q and -Q only
    bases = ctx.load_bases(pts, window_bits=c)
    exp, einf = oracle.msm(pts, s)
    assert not einf
    out, inf = ctx.msm(bases, s)
    assert not inf and (out == exp).all()
    # in a batch between two members that are the identity (P and -P, Q and -Q in one bucket each)
    s2 = oracle.ints_to_array([1, 1, L + 1, L + 1])
    out, inf = msm_batch(ctx, bases, np.stack([s2, s, s2]), 4)
    assert inf == [True, False, True] and (out[1] == exp).all()


def test_heavy_bucket_in_batch(ctx, oracle):
    """c = 17: 2081 entries in bucket 4 is more than 64 segments of 32, so that bucket's sum comes from the heavy combine
    while the others of the same batch are read from their segment sums."""
    c, n = 17, 2300
    pts = oracle.known_dlog_bases(SEED, n)
    heavy = oracle.splitmix_fr(0x4EA7, n, False)
    heavy[:md.SEG_LEN * (md.COMBINE_SEQ + 1) + 1] = oracle.int_to_limbs(5)
    counts = md.bucket_counts_np(heavy, c)
    assert md.is_heavy(counts[4]) and int((counts >= md.HEAVY_MIN).sum()) == 1
    bases = ctx.load_bases(pts, window_bits=c)
    rng = random.Random(0x4EA7)
    vectors = np.stack([oracle.splitmix_fr(0x100 + i, n, False) for i in range(2)] + [heavy] +
                       [oracle.ints_to_array([rng.randrange(R) for _ in range(n)]), heavy])
    out, inf = msm_batch(ctx, bases, vectors, n + 1)
    for b in range(vectors.shape[0]):
        exp, einf = oracle.msm(pts, vectors[b])
        assert inf[b] == einf and (out[b] == exp).all(), b
    exp, _ = oracle.msm(pts, heavy)
    out, inf = rb.VariableBaseMSM.msm_bigint(ctx, bases, heavy)
    assert not inf and (out == exp).all()
