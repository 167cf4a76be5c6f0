"""The claims of `pairing_cases.py` and the host pairing against them, without a GPU: the independent pure-Python
pairing agrees with the bilinearity prediction on a small sample; the host `b200_pairing_check` gives the predicted
verdict on every algebraic case for m = 1 … 8 pairs over seeded G2 points, H, -H, a repeated point and the identity
record; its verdicts on a twist point outside the r-torsion are recorded; G1 records off the curve or with a coordinate
moved to v + q are refused in any slot."""
import time

import numpy as np
import pytest

import bn254_pairing_py as pr
import bn254_py as py
import pairing_cases as pc
from renegade_b200 import _lib
from renegade_b200.backend import g2_in_subgroup, pairing_check


@pytest.fixture(scope="module")
def pts(oracle, g2_raw):
    return pc.Points(g2_raw[0])


def host(g1, g2) -> np.ndarray:
    """b200_pairing_check of every check: g1 (n, m, 8), g2 (m, 16)"""
    return np.array([pairing_check(list(c), list(g2)) if len(g2) else True for c in g1], dtype=bool)


def mismatches(got, want) -> list:
    return [c for c in range(len(want)) if bool(got[c]) != bool(want[c])]


# ---- the builder's own claims ------------------------------------------------------------------------------------------
def test_points_are_what_they_claim(pts, g2_raw, oracle):
    assert (pts.g2(1) == g2_raw[0]).all()
    h = pr.decode_g2_mont(g2_raw[0].tobytes(), 0)
    neg_h = (h[0], ((-h[1][0]) % pr.Q, (-h[1][1]) % pr.Q))
    assert pts.g2(pr.R - 1).tobytes() == pr.encode_g2_mont(neg_h)
    assert not pts.g2(0).any()
    for b in pc.g2_scalars(8, "distinct") + [1, pr.R - 1]:
        assert pr.g2_is_on_curve(pr.decode_g2_mont(pts.g2(b).tobytes(), 0)) and g2_in_subgroup(pts.g2(b))
    a = 0x1234567890ABCDEF1234567890ABCDEF
    assert (pts.g1(1) == pc.G1_GEN).all() and not pts.g1(0).any()
    assert oracle.g1_on_curve(pts.g1(a))
    assert (pts.g1(a + 1) == oracle.g1_add(pts.g1(a), 0, pc.G1_GEN, 0)[0]).all()  # the addition shortcut
    assert (pts.g1(pr.R - a) == oracle.g1_mul(pc.G1_GEN, 0, oracle.int_to_limbs(pr.R - a))[0]).all()  # -P
    assert py.decode_g1_mont(pts.g1(pr.R - a).tobytes(), 0)[1] == (-py.decode_g1_mont(pts.g1(a).tobytes(), 0)[1]) % pr.Q


@pytest.mark.parametrize("m", range(1, pc.MAX_PAIRS + 1))
def test_sweeps_and_edge_rows_hold_and_fail_as_claimed(pts, m):
    for kind in ("distinct", "edges", "identity"):
        b = pc.g2_scalars(m, kind)
        assert len(b) == m
        if kind == "distinct":
            assert len(set(b)) == m and not {0, 1, pr.R - 1} & set(b)
        s = pc.Sweep(pts, b, 200)
        assert s.predicted(s.hold).all()
        live = [j for j in range(m) if b[j]]
        if live:
            assert not s.predicted(s.fail).any()
            broken = {next(j for j in range(m) if h[j] != f[j]) for h, f in zip(s.hold, s.fail)}
            assert broken == set(live), (kind, broken)  # every live slot is the broken one somewhere
        for n in (1, 63, 64, 65, 129, 200):
            for name, bad in pc.placements(n).items():
                assert list(np.flatnonzero(~s.predicted(s.rows(n, bad) if live else s.hold[:n]))) == \
                    (sorted(bad) if live else []), (kind, n, name)
        rows = pc.edge_rows(b, 64)
        v = [pc.holds(a, b) for a in rows]
        assert any(v) and (not live or not all(v))


# ---- the independent pairing ------------------------------------------------------------------------------------------
def test_python_pairing_agrees_with_the_prediction(pts):
    """one holding and one failing check for m = 1, 2 and 8 over distinct seeded G2 points, on the pure-Python
    optimal-ate pairing (≈ 2.5 s on one x86-64 core)"""
    t0 = time.time()
    for m in (1, 2, 8):
        b = pc.g2_scalars(m, "distinct", seed=1)
        s = pc.Sweep(pts, b, 4, seed=1)
        for rows, want in ((s.hold[:1], True), (s.fail[:1], False)):
            assert s.predicted(rows).tolist() == [want]
            g1 = s.g1(rows)[0]
            pairs = []
            for j in range(m):
                p = py.decode_g1_mont(g1[j].tobytes(), 0)
                pairs.append((None if p == (0, 0) else p, pr.decode_g2_mont(s.g2[j].tobytes(), 0)))
            assert pr.pairing_product_is_one(pairs) == want, (m, want)
            assert pairing_check(list(g1), list(s.g2)) == want, (m, want)
    print("pure-Python pairing sample: %.1f s" % (time.time() - t0))


# ---- the host pairing on every algebraic case ------------------------------------------------------------------------
@pytest.mark.parametrize("m", range(1, pc.MAX_PAIRS + 1))
def test_host_pairing_gives_the_predicted_verdicts(pts, m):
    for kind in ("distinct", "edges", "identity"):
        b = pc.g2_scalars(m, kind)
        g2 = np.stack([pts.g2(x) for x in b])
        s = pc.Sweep(pts, b, 12)
        rows = s.hold + s.fail + pc.edge_rows(b, 24)
        want = np.array([pc.holds(a, b) for a in rows])
        got = host(pc.g1_records(pts, rows, m), g2)
        assert not mismatches(got, want), (m, kind, mismatches(got, want))


def test_identity_g2_record_contributes_one(pts):
    b = pc.g2_scalars(3, "distinct")
    s = pc.Sweep(pts, b, 8)
    g2 = np.stack([pts.g2(x) for x in b])
    for c in range(8):
        for rows in (s.hold, s.fail):
            g1 = s.g1([rows[c]])[0]
            want = pairing_check(list(g1), list(g2))
            # a fourth pair against the identity record, whatever its G1 point: the verdict stays
            for extra in (pc.G1_GEN, pts.g1(0xABCDEF), pc.G1_IDENTITY):
                assert pairing_check(list(g1) + [extra], list(g2) + [pc.G2_IDENTITY]) == want
    assert pairing_check([pc.G1_GEN], [pc.G2_IDENTITY]) and pairing_check([pc.G1_GEN] * 8, [pc.G2_IDENTITY] * 8)
    assert not pairing_check([pc.G1_GEN], [pts.g2(1)])


@pytest.mark.parametrize("m,n", pc.TWIST_CASES)
def test_host_verdicts_on_a_twist_point_outside_the_subgroup(pts, m, n):
    case = pc.TwistCase(pts, m, n)
    assert not g2_in_subgroup(case.g2[case.t])
    got = host(case.g1, case.g2)
    assert got.tolist() == case.recorded(), mismatches(got, case.recorded())
    assert any(v is None for v in case.verdicts) and any(case.verdicts)


# ---- refused G1 records ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("m", [1, 4, 8])
def test_host_refuses_g1_records_outside_the_curve_or_the_field(pts, m):
    b = pc.g2_scalars(m, "distinct")
    s = pc.Sweep(pts, b, 1)
    g2 = list(s.g2)
    g1 = s.g1(s.hold[:1])[0]
    g1[0] = pts.g1(0x5A5A5A)
    for j in sorted({0, m // 2, m - 1}):
        for bad in (pc.off_curve(g1[j] if g1[j].any() else pc.G1_GEN), pc.plus_q(g1[j], 0), pc.plus_q(g1[j], 1)):
            rows = g1.copy()
            rows[j] = bad
            with pytest.raises(_lib.B200Error) as err:
                pairing_check(list(rows), g2)
            assert err.value.code == _lib.B200_ERR_NOT_ON_CURVE, (m, j)
