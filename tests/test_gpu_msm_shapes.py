"""GPU: the MSM's bucket pipeline at the shapes where it can go wrong, against the oracle (bit-exact after affine
normalisation) and, at 2^17 points, the known-discrete-log closed form.

Uniform random scalars almost never reach these paths, so every test builds its digits on purpose and asserts, with the
Python restatement of the recoding (tests/msm_digits.py), that its input has the shape it is about — exact bucket
counts, more heavy buckets than the combine grid has blocks, the edge digits — so that a change of the kernel's
constants cannot turn a test into one that passes without reaching its path:
  * the signed-digit recoding at every window width 8 ... 23: digits half, half + 1 and 2^c (magnitude 0, carry only),
    carry chains through every window, 2^m +- 1 at window boundaries, r - 1; canonical and Montgomery scalars;
  * buckets of exactly 1, 31, 32, 33, 63, 64, 65, 2047, 2048, 2049, 2080 and 2081 entries around the segment length
    (32) and the heavy threshold (64 segments), positive and negative digits in one bucket, P and -P in one bucket
    (running sums through the identity), a heavy bucket whose total is the identity;
  * more heavy buckets than the grid-stride combine kernel has blocks (4 per SM), so blocks take a second bucket;
  * batched MSMs whose first, middle or last member is the identity, one that cancels, the heavy vector, and a batch
    at c = 20 whose bucket histogram spans hundreds of scan tiles;
  * base_off + n = number of bases, n = 1 included."""
import ctypes as C
import os
import random

import numpy as np
import pytest

import msm_digits as md
import renegade_b200 as rb

pytestmark = pytest.mark.gpu

R = md.R
Q = 0x30644E72E131A029B85045B68181585D97816A916871CA8D3C208C16D87CFD47
SEED = 0xB200


@pytest.fixture(params=[False, True], ids=["latency", "throughput"])
def mode(request, ctx):
    """Both MSM tunings (b200_msm_tuning); results must be identical."""
    ctx.msm_tuning(request.param)
    yield request.param
    ctx.msm_tuning(False)


def ints(a: np.ndarray) -> list[int]:
    return [x | y << 64 | z << 128 | w << 192 for x, y, z, w in np.asarray(a, dtype=np.uint64).reshape(-1, 4).tolist()]


def negate(pts: np.ndarray) -> np.ndarray:
    """-P for affine points x || y (Montgomery): y -> q - y."""
    out = pts.copy()
    for i, y in enumerate(ints(pts[:, 4:])):
        assert y, "identity rows are not negated"
        out[i, 4:] = [((Q - y) >> (64 * k)) & ((1 << 64) - 1) for k in range(4)]
    return out


def sm_count() -> int:
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def msm_batch(ctx, bases, vectors: np.ndarray, stride: int):
    """b200_msm_batch_device over `vectors` (batch, n, 4) canonical scalars laid out `stride` apart on the device."""
    import torch
    from renegade_b200 import _lib
    batch, n = vectors.shape[0], vectors.shape[1]
    s = np.full((batch, stride, 4), 0xA5A5A5A5A5A5A5A5, dtype=np.uint64)  # the gaps must not be read
    s[:, :n] = vectors
    t = torch.from_numpy(s.view(np.int64)).cuda()
    torch.cuda.synchronize()
    out = np.zeros((batch, 8), dtype=np.uint64)
    inf = (C.c_int * batch)()
    _lib.check(ctx._lib.b200_msm_batch_device(ctx._h, bases._h, 0, C.c_void_p(t.data_ptr()), n, stride, batch, 0,
                                              out.ctypes.data_as(C.c_void_p), inf))
    return out, [bool(v) for v in inf]


def cancelling(a: list[int], rng: random.Random) -> list[int]:
    """Scalars s with sum a_i s_i = 0 mod r (random but for s_0), for bases a_i G."""
    s = [0] + [rng.randrange(R) for _ in a[1:]]
    s[0] = -sum(x * y for x, y in zip(a[1:], s[1:])) * pow(a[0], -1, R) % R
    return s


# ---- recoding edges ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def pts320(oracle):
    return oracle.known_dlog_bases(SEED, 320)


@pytest.mark.parametrize("c", range(8, 24))
def test_recoding_edges_every_window_width(ctx, oracle, pts320, mode, c):
    pts, n = pts320, pts320.shape[0]
    half = 1 << (c - 1)
    edges = md.edge_scalars(c)
    rng = random.Random(0xED6E + c)
    vals = edges + [rng.randrange(R) for _ in range(-len(edges) % n)]
    raws, chain = set(), False
    for s in edges:
        digits, carry = md.signed_digits(s, c)
        assert carry == 0
        raws |= {raw for _, raw, _, _ in digits}
        chain |= all(d[1] >= (1 << c) - 1 for d in digits[:-1])
    assert {half, half + 1, 1 << c} <= raws and chain  # the edge digits and a carry through every window occur
    bases = ctx.load_bases(pts, window_bits=c)
    assert bases.plan == {"window_bits": c, "digits": md.num_windows(c), "physical_windows": 1,
                          "tables": md.num_windows(c)}
    for k in range(0, len(vals), n):
        s = oracle.ints_to_array(vals[k:k + n])
        exp, einf = oracle.msm(pts, s)
        out, inf = rb.VariableBaseMSM.msm_bigint(ctx, bases, s)
        assert inf == einf and (out == exp).all(), (c, k)
        out, inf = rb.UnivariateKzgPCS.commit(ctx, bases, oracle.array_to_mont(oracle.FR, s))
        assert inf == einf and (out == exp).all(), (c, k, "montgomery")


# ---- bucket occupancy ---------------------------------------------------------------------------------------------
S, K = md.SEG_LEN, md.COMBINE_SEQ
COUNTS = [1, S - 1, S, S + 1, 2 * S - 1, 2 * S, 2 * S + 1, S * K - 1, S * K, S * K + 1, S * (K + 1), S * (K + 1) + 1]


def test_bucket_occupancy_boundaries(ctx, oracle, mode):
    """c = 12, small digits d < 2^11: bucket d - 1 holds exactly the chosen number of entries.  Entries land in a bucket
    in atomic order, which varies from run to run; three runs must all equal the oracle."""
    c = 12
    top = 1 << c
    rows, scal = [], []  # (points, scalars) blocks
    fresh = oracle.known_dlog_bases(SEED, sum(COUNTS) + 65 + 2049 + 1040 + 2)
    used = 0

    def take(k):
        nonlocal used
        used += k
        return fresh[used - k:used]

    for j, k in enumerate(COUNTS):  # magnitudes 16 ... 27, positive digits
        rows.append(take(k))
        scal += [16 + j] * k
    for d, pos, neg in ((100, 40, 25), (101, 1000, S * K + 1 - 1000)):  # +d and -d (scalar 2^c - d) in one bucket
        rows.append(take(pos + neg))
        scal += [d] * pos + [top - d] * neg
    pm = take(1040)  # 1040 pairs P, -P: a heavy bucket whose total is the identity
    rows += [pm, negate(pm)]
    scal += [300] * 2080
    one = take(2)  # one point P and -P repeated: running sums keep passing through the identity and doubling
    rows += [np.repeat(one[:1], 17, axis=0), np.repeat(negate(one[:1]), 16, axis=0),
             np.repeat(one[1:], 32, axis=0), np.repeat(negate(one[1:]), 32, axis=0)]
    scal += [301] * 33 + [302] * 64
    pts = np.concatenate(rows)
    perm = np.random.default_rng(12).permutation(pts.shape[0])  # interleave the blocks in index order
    pts, scal = pts[perm], [scal[i] for i in perm]
    s = oracle.ints_to_array(scal)

    counts = md.bucket_counts_np(s, c)
    for j, k in enumerate(COUNTS):
        assert counts[16 + j - 1] == k
    assert counts[99] == 65 and counts[100] == S * K + 1 and counts[299] == 2080 and counts[300] == 33 and counts[301] == 64
    assert [md.is_heavy(counts[b]) for b in (16 + 7 - 1, 16 + 8 - 1, 16 + 9 - 1, 100, 299)] == [False, False, True, True, True]

    bases = ctx.load_bases(pts, window_bits=c)
    assert bases.plan["window_bits"] == c and bases.plan["physical_windows"] == 1
    exp, einf = oracle.msm(pts, s)
    assert not einf
    for _ in range(3):
        out, inf = ctx.msm(bases, s)
        assert inf == einf and (out == exp).all()
    out, inf = ctx.msm(bases, oracle.array_to_mont(oracle.FR, s), montgomery=True)
    assert inf == einf and (out == exp).all()
    # the P / -P buckets alone: the MSM is the identity
    only = oracle.ints_to_array([v if v in (300, 302) else 0 for v in scal])
    out, inf = ctx.msm(bases, only)
    assert inf and not out.any()


# ---- heavy buckets beyond the combine grid --------------------------------------------------------------------------
HEAVY_N = 1 << 17


@pytest.fixture(scope="module")
def heavy_bases(ctx, oracle):
    """2^17 known-discrete-log bases a_i G at c = 8 with every window in its own bucket range (32 physical windows):
    32 x 128 buckets, so digits drawn from 40 values make ~1280 buckets of ~3300 entries."""
    import torch
    d_pts = torch.empty((HEAVY_N, 8), dtype=torch.int64, device="cuda")
    torch.cuda.synchronize()
    ctx.known_dlog_bases_device(SEED, HEAVY_N, d_pts.data_ptr())
    old = os.environ.get("B200_MSM_PHYS_WINDOWS")
    os.environ["B200_MSM_PHYS_WINDOWS"] = "32"
    try:
        bases = ctx.load_bases_device(d_pts.data_ptr(), HEAVY_N, window_bits=8)
    finally:
        if old is None:
            del os.environ["B200_MSM_PHYS_WINDOWS"]
        else:
            os.environ["B200_MSM_PHYS_WINDOWS"] = old
    assert bases.plan == {"window_bits": 8, "digits": 32, "physical_windows": 32, "tables": 1}
    pts = d_pts.cpu().numpy().view(np.uint64)
    assert (pts[:64] == oracle.known_dlog_bases(SEED, 64)).all()
    return bases, pts, ints(oracle.splitmix_fr(SEED, HEAVY_N, False))


def heavy_scalars(negative: bool) -> np.ndarray:
    """Every byte from {1 ... 40}, or (negative) bytes 0 ... 30 from {216 ... 255}: negative digits of magnitude
    1 ... 40 whose carries move the next window's digit by one.  The top byte stays <= 40, so s < r."""
    rng = np.random.default_rng(0x4EA7 + negative)
    b = rng.integers(1, 41, size=(HEAVY_N, 32), dtype=np.uint8)
    if negative:
        b[:, :31] = rng.integers(216, 256, size=(HEAVY_N, 31), dtype=np.uint8)
    return b.view(np.uint64).reshape(HEAVY_N, 4).copy()


def closed_form(oracle, pyoracle, a: list[int], s: np.ndarray):
    k = sum(x * y for x, y in zip(a, ints(s))) % R
    g = np.frombuffer(pyoracle.encode_g1_mont(pyoracle.G1_GEN), dtype=np.uint64)
    return oracle.g1_mul(g, False, oracle.int_to_limbs(k))


@pytest.mark.parametrize("negative", [False, True], ids=["positive", "negative"])
def test_more_heavy_buckets_than_combine_blocks(ctx, oracle, pyoracle, heavy_bases, mode, negative):
    bases, pts, a = heavy_bases
    s = heavy_scalars(negative)
    counts = md.bucket_counts_np(s, 8, n_phys=32)
    heavy = int((counts >= md.HEAVY_MIN).sum())
    assert heavy > 4 * sm_count(), heavy  # blocks of the grid-stride combine go round at least twice
    assert int(s.view(np.uint8).reshape(HEAVY_N, 32)[:, 31].max()) <= 40 and 41 << 248 < R  # canonical scalars
    exp, einf = oracle.msm(pts, s)
    cf, cinf = closed_form(oracle, pyoracle, a, s)
    assert not einf and not cinf and (exp == cf).all()
    out, inf = ctx.msm(bases, s)
    assert not inf and (out == exp).all()


# ---- batched MSM epilogue ---------------------------------------------------------------------------------------------
def test_batch_with_identity_members_and_heavy_vector(ctx, oracle, heavy_bases):
    """One field inversion serves the whole batch (Montgomery's trick over the members that are not the identity):
    identity members first, in the middle and last, a vector that cancels, the heavy vector and random vectors."""
    bases, pts, a = heavy_bases
    rng = random.Random(0xBA7C)
    zero = np.zeros((HEAVY_N, 4), dtype=np.uint64)
    rand = [oracle.splitmix_fr(0x100 + i, HEAVY_N, False) for i in range(2)]
    cancel = oracle.ints_to_array(cancelling(a, rng))
    vectors = np.stack([zero, rand[0], cancel, zero, heavy_scalars(False), rand[1], zero])
    exp = [oracle.msm(pts, v) for v in vectors]
    assert [e[1] for e in exp] == [True, False, True, True, False, False, True]
    heavy = int((md.bucket_counts_np(vectors[4], 8, n_phys=32) >= md.HEAVY_MIN).sum())
    assert heavy > 4 * sm_count()
    out, inf = msm_batch(ctx, bases, vectors, HEAVY_N + 8)
    for b, (e, einf) in enumerate(exp):
        assert inf[b] == einf and (out[b] == e).all(), b


def test_batch_across_many_scan_tiles(ctx, oracle):
    """c = 20: 2^19 buckets per MSM, so the batch's bucket histogram spans hundreds of tiles of the single-pass scan,
    with the members' ranges side by side."""
    n, c = 3000, 20
    pts = oracle.known_dlog_bases(SEED, n)
    a = ints(oracle.splitmix_fr(SEED, n, False))
    bases = ctx.load_bases(pts, window_bits=c)
    assert bases.plan["window_bits"] == c and bases.plan["physical_windows"] == 1
    rng = random.Random(0x5CA7)
    zero = np.zeros((n, 4), dtype=np.uint64)
    edges = md.edge_scalars(c)[:n]
    vectors = np.stack([zero, oracle.splitmix_fr(0x200, n, False), oracle.ints_to_array(cancelling(a, rng)), zero,
                        oracle.ints_to_array(edges + [0] * (n - len(edges))), zero])
    tiles = vectors.shape[0] * (1 << (c - 1)) // md.SCAN_TILE
    assert tiles >= 500, tiles
    exp = [oracle.msm(pts, v) for v in vectors]
    assert [e[1] for e in exp] == [True, False, True, True, False, True]
    out, inf = msm_batch(ctx, bases, vectors, n + 5)
    for b, (e, einf) in enumerate(exp):
        assert inf[b] == einf and (out[b] == e).all(), b


# ---- base offset at the end of the bases ----------------------------------------------------------------------------
@pytest.mark.parametrize("window_bits", [0, 9])
def test_base_off_at_the_tail(ctx, oracle, window_bits):
    from renegade_b200._lib import B200Error
    n = 700
    pts = oracle.known_dlog_bases(SEED, n)
    bases = ctx.load_bases(pts, window_bits=window_bits)
    for off in (0, 1, 350, n - 2, n - 1):
        m = n - off
        s = oracle.splitmix_fr(0x7A11 + off, m, False)
        exp, einf = oracle.msm(pts[off:], s)
        out, inf = ctx.msm(bases, s, base_off=off)
        assert inf == einf and (out == exp).all(), off
    # the last base alone, with the scalar r - 1: -P
    out, inf = ctx.msm(bases, oracle.ints_to_array([R - 1]), base_off=n - 1)
    assert not inf and (out == negate(pts[n - 1:])[0]).all()
    with pytest.raises(B200Error):
        ctx.msm(bases, oracle.splitmix_fr(1, 2, False), base_off=n - 1)
