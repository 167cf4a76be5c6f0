"""Many pairing checks on the device (`b200_pairing_check_many`, `backend.pairing_check_many`): every answer must equal
the host pairing's (`b200_pairing_check`) over the same pairs, and a few equal the pure-Python pairing's.  The points
are the reference's SRS head (its first 512 G1 powers tau^i G and its G2 pair H, tau H)."""
import ctypes as C
import random

import numpy as np
import pytest

import renegade_b200 as rb
from renegade_b200 import _lib
from renegade_b200.backend import pairing_check, pairing_check_many

pytestmark = pytest.mark.gpu

Q = 21888242871839275222246405745257275088696311157297823662689037894645226208583  # the base field modulus
IDENTITY = np.zeros(8, dtype=np.uint64)


def _neg(pt):
    """-P for a 64-byte Montgomery record (the Montgomery form of -y is q - (that of y))."""
    y = int.from_bytes(np.asarray(pt[4:8], dtype="<u8").tobytes(), "little")
    out = np.array(pt, dtype=np.uint64).copy()
    out[4:8] = np.frombuffer(((Q - y) % Q).to_bytes(32, "little"), dtype="<u8")
    return out


@pytest.fixture(scope="module")
def pts(ctx, srs_head):
    return rb.parse_ptau_file(ctx, srs_head, count=512).powers_of_g_host


def _host(g1, g2):
    """b200_pairing_check of every check: g1 (n, m, 8), g2 (m, 16)."""
    return np.array([pairing_check(list(c), list(g2)) if len(g2) else True for c in g1], dtype=bool)


def _ratio_checks(pts, step):
    """e(P_i, tau H) e(-P_{i+step_i}, H) for i < 511 (the reference's SRS test with step 1)"""
    return np.stack([np.stack([pts[i], _neg(pts[min(i + step(i), 511)])]) for i in range(511)])


def test_srs_ratio_checks_all_hold(ctx, pts, g2_raw):
    h, tau_h = g2_raw
    g2 = np.stack([tau_h, h])
    g1 = _ratio_checks(pts, lambda i: 1)
    got = pairing_check_many(ctx, g2, g1)
    assert got.shape == (511,) and got.all()
    assert (got == _host(g1, g2)).all()


def test_skipped_power_fails_exactly_there(ctx, pts, g2_raw):
    h, tau_h = g2_raw
    g2 = np.stack([tau_h, h])
    bad = {0, 17, 255, 508}
    g1 = _ratio_checks(pts, lambda i: 2 if i in bad else 1)
    got = pairing_check_many(ctx, g2, g1)
    assert [i for i in range(511) if not got[i]] == sorted(bad)
    assert (got == _host(g1, g2)).all()


def test_against_the_python_pairing(ctx, pts, g2_raw, pyoracle):
    import bn254_pairing_py as pr
    py = pyoracle
    h, tau_h = g2_raw
    g2 = np.stack([tau_h, h])
    g1 = np.stack([np.stack([pts[3], _neg(pts[4])]), np.stack([pts[3], _neg(pts[5])])])
    got = pairing_check_many(ctx, g2, g1)
    raw = h.tobytes() + tau_h.tobytes()
    qh, qt = pr.decode_g2_mont(raw, 0), pr.decode_g2_mont(raw, 1)
    for c in range(2):
        a, b = (py.decode_g1_mont(g1[c, j].tobytes(), 0) for j in range(2))
        assert got[c] == pr.pairing_product_is_one([(a, qt), (b, qh)])
    assert got.tolist() == [True, False]


@pytest.mark.parametrize("m", [1, 2, 3, 4])
def test_pair_counts_identities_and_repeated_g2(ctx, pts, g2_raw, m):
    """Checks of m pairs over (tau H, H) repeated, with identity G1 points and products that hold or fail."""
    h, tau_h = g2_raw
    rnd = random.Random(m)
    g2 = np.stack([tau_h if j % 2 == 0 else h for j in range(m)])
    checks = []
    for c in range(24):
        row = [IDENTITY if rnd.randrange(4) == 0 else pts[rnd.randrange(512)] for _ in range(m)]
        if c % 3 == 0 and m >= 2:  # a product that holds: ratio pairs, identities elsewhere
            i = rnd.randrange(510)
            row = [IDENTITY] * m
            row[0], row[1] = pts[i], _neg(pts[i + 1])
        if c % 5 == 1:
            row = [IDENTITY] * m  # every pair contributes 1
        checks.append(np.stack(row))
    g1 = np.stack(checks)
    got = pairing_check_many(ctx, g2, g1)
    want = _host(g1, g2)
    assert (got == want).all()
    assert want.any() and not want.all()


def test_no_checks_and_no_pairs(ctx, g2_raw, pts):
    h, tau_h = g2_raw
    g2 = np.stack([tau_h, h])
    assert pairing_check_many(ctx, g2, np.zeros((0, 2, 8), dtype=np.uint64)).shape == (0,)
    assert pairing_check_many(ctx, np.zeros((0, 16), dtype=np.uint64), np.zeros((3, 0, 8), dtype=np.uint64)).all()


def test_null_arguments(ctx, g2_raw, pts):
    lib = ctx._lib
    h, tau_h = g2_raw
    g2 = np.stack([tau_h, h])
    g1 = np.stack([pts[0], _neg(pts[1])])
    out = (C.c_uint8 * 1)()
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    assert lib.b200_pairing_check_many(None, p(g2), 2, p(g1), 1, out) == _lib.B200_ERR_INVALID
    assert lib.b200_pairing_check_many(ctx._h, None, 2, p(g1), 1, out) == _lib.B200_ERR_INVALID
    assert lib.b200_pairing_check_many(ctx._h, p(g2), 2, None, 1, out) == _lib.B200_ERR_INVALID
    assert lib.b200_pairing_check_many(ctx._h, p(g2), 2, p(g1), 1, None) == _lib.B200_ERR_INVALID
    many = np.stack([tau_h] * 9)
    assert lib.b200_pairing_check_many(ctx._h, p(many), 9, p(np.zeros((9, 8), dtype=np.uint64)), 1,
                                       out) == _lib.B200_ERR_INVALID
    assert lib.b200_pairing_check_many(ctx._h, p(g2), 2, p(g1), 1, out) == _lib.B200_OK and out[0] == 1


def test_points_off_the_curve(ctx, pts, g2_raw):
    h, tau_h = g2_raw
    g2 = np.stack([tau_h, h])
    g1 = _ratio_checks(pts, lambda i: 1)[:8].copy()
    off = g1.copy()
    off[5, 1, 0] ^= np.uint64(1)  # x moved: off the curve
    x = int.from_bytes(g1[6, 0, 0:4].tobytes(), "little")
    non_canonical = g1.copy()
    non_canonical[6, 0, 0:4] = np.frombuffer((x + Q).to_bytes(32, "little"), dtype="<u8")  # x + q: outside [0, q)
    for bad, c in ((off, 5), (non_canonical, 6)):
        with pytest.raises(_lib.B200Error) as err:
            pairing_check_many(ctx, g2, bad)
        assert err.value.code == _lib.B200_ERR_NOT_ON_CURVE
        assert "check %d" % c in str(err.value)
        with pytest.raises(_lib.B200Error) as err:
            pairing_check(list(bad[c]), list(g2))  # the host check refuses the same pairs
        assert err.value.code == _lib.B200_ERR_NOT_ON_CURVE
    both = off.copy()
    both[6] = non_canonical[6]
    with pytest.raises(_lib.B200Error) as err:
        pairing_check_many(ctx, g2, both)
    assert "check 5" in str(err.value)  # the first such check
    bad_g2 = g2.copy()
    bad_g2[1, 0] ^= np.uint64(1)
    with pytest.raises(_lib.B200Error) as err:
        pairing_check_many(ctx, bad_g2, g1)
    assert err.value.code == _lib.B200_ERR_NOT_ON_CURVE and "G2 point 1" in str(err.value)
