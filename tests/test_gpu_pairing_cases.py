"""The device pairing held to bilinearity (`pairing_cases.py`): `b200_pairing_check_many` at every pair count m = 0 … 8,
on G2 points b H other than the SRS pair, over 1 … 4097 checks with the failing checks placed around the kernel's
64-thread blocks, gives exactly the verdicts predicted with Python integers, and the host pairing's on every check up
to 129 and on a seeded sample above; twist points outside the r-torsion give the host's verdicts; refused G1 records deep
in a batch are named.  The verifiers do not hard-wire the G2 generator: under (kH, k tau H) `b200_plonk_verify_each`,
`b200_plonk_batch_verify` and `b200_srs_check` (its locate pass, `k_srs_pairs`) give what they give under (H, tau H)."""
import random

import numpy as np
import pytest

import bn254_pairing_py as pr
import bn254_py as py
import pairing_cases as pc
import renegade_b200 as rb
from renegade_b200 import _lib, synth
from renegade_b200.backend import (PlonkKzgSnark, VerifyingKey, link_proofs, pairing_check, pairing_check_many,
                                   verify_link_proof)
from test_gpu_batch_verify import LAYOUT, LINK_VALS, SPECS, Env, _tamper, proof_items
from test_gpu_srs_check import OTHER_TAU, check, expected_pairs, g1_dbl, g1_neg, seeded_points

pytestmark = pytest.mark.gpu

NS = [1, 63, 64, 65, 127, 128, 129, 1000, 4097]
HOST_ALL = 129     # batches up to this size are compared with the host pairing check by check
HOST_SAMPLE = 16   # checks of each larger batch compared with the host pairing
G2_K = 0x3A5F00D1E2C3B4A5968778695A4B3C2D1E0F  # the seeded k of the second G2 pair (kH, k tau H)
R = pc.R


@pytest.fixture(scope="module")
def pts(oracle, g2_raw):
    return pc.Points(g2_raw[0])


class HostCache:
    """b200_pairing_check of rows of G1 scalars over one set of G2 points, each distinct row once"""

    def __init__(self, pts, g2):
        self.pts, self.g2, self.seen = pts, g2, {}

    def __call__(self, row) -> bool:
        key = tuple(row)
        if key not in self.seen:
            g1 = pc.g1_records(self.pts, [row], len(row))[0]
            self.seen[key] = pairing_check(list(g1), list(self.g2)) if len(row) else True
        return self.seen[key]


def assert_same(got, want, what: str, m: int, against: str = "predicted"):
    got, want = np.asarray(got, dtype=bool), np.asarray(want, dtype=bool)
    bad = np.flatnonzero(got != want)
    assert got.shape == want.shape and not bad.size, "m = %d, %s: device != %s at check(s) %s (device %s, %s %s)" % (
        m, what, against, bad[:12].tolist(), got[bad[:12]].astype(int).tolist(), against,
        want[bad[:12]].astype(int).tolist())


# ---- b200_pairing_check_many against bilinearity ---------------------------------------------------------------------
@pytest.mark.parametrize("m", range(0, pc.MAX_PAIRS + 1))
def test_every_pair_count_batch_size_and_failing_position(ctx, pts, m):
    """m seeded, distinct G2 points; for each n of NS the failing checks none, first, at 63 / 64 / 65, last,
    alternating and everywhere: device = prediction exactly, = host on every check up to 129 and on a sample above"""
    b = pc.g2_scalars(m, "distinct")
    s = pc.Sweep(pts, b, max(NS))
    host = HostCache(pts, s.g2)
    rng = random.Random(0xC0FFEE + m)
    for n in NS:
        for name, bad in pc.placements(n).items():
            if m == 0 and bad:
                continue  # no pairs: every check holds
            rows = s.rows(n, bad)
            want = s.predicted(rows)
            assert want.tolist() == [c not in bad for c in range(n)]
            got = pairing_check_many(ctx, s.g2, s.g1(rows))
            what = "n = %d, failing %s" % (n, name)
            assert_same(got, want, what, m)
            idx = list(range(n)) if n <= HOST_ALL else sorted(rng.sample(range(n), HOST_SAMPLE))
            assert_same(got[idx], [host(rows[c]) for c in idx], what + " (checks %s)" % idx[:4], m, "host")


@pytest.mark.parametrize("m", range(1, pc.MAX_PAIRS + 1))
@pytest.mark.parametrize("kind", ["edges", "identity"])
def test_g2_edges_and_g1_edges(ctx, pts, m, kind):
    """G2 points H, -H, one point in two slots (edges) or the identity record in a slot (identity); checks of every
    holding kind, failing twins at every slot, one G1 point in all m slots, P and -P: device = prediction = host"""
    b = pc.g2_scalars(m, kind)
    g2 = np.stack([pts.g2(x) for x in b])
    rows = pc.edge_rows(b, 129 if kind == "edges" else 65, seed=m)
    want = np.array([pc.holds(a, b) for a in rows])
    got = pairing_check_many(ctx, g2, pc.g1_records(pts, rows, m))
    assert_same(got, want, "%s G2 points" % kind, m)
    host = HostCache(pts, g2)
    assert_same(got, [host(a) for a in rows], "%s G2 points" % kind, m, "host")


def test_every_g2_record_the_identity(ctx, pts):
    for m in (1, 8):
        g1 = pc.g1_records(pts, [[random.Random(c).randrange(R) for _ in range(m)] for c in range(70)], m)
        assert pairing_check_many(ctx, np.zeros((m, 16), dtype=np.uint64), g1).all()


@pytest.mark.parametrize("m,n", pc.TWIST_CASES)
def test_twist_point_outside_the_subgroup(ctx, pts, m, n):
    """no algebraic verdict where a G1 point meets the twist point: device = host on every check, = the recorded
    verdicts (`test_pairing_cases_cpu.py`)"""
    case = pc.TwistCase(pts, m, n)
    got = pairing_check_many(ctx, case.g2, case.g1)
    assert_same(got, case.recorded(), "twist point in slot %d" % case.t, m, "recorded")
    host = np.array([pairing_check(list(c), list(case.g2)) for c in case.g1])
    assert_same(got, host, "twist point in slot %d" % case.t, m, "host")


@pytest.mark.parametrize("m", [1, 3, 8])
def test_refused_g1_records_deep_in_a_large_batch(ctx, pts, m):
    b = pc.g2_scalars(m, "distinct")
    s = pc.Sweep(pts, b, 4097)
    rows = s.rows(4097, set(range(0, 4097, 7)))
    g1 = s.g1(rows)
    j = m - 1
    live = g1[:, j].any(axis=1)

    def refused(bad: dict, first: int):
        x = g1.copy()
        for c, rec in bad.items():
            x[c, j] = rec
        with pytest.raises(_lib.B200Error) as err:
            pairing_check_many(ctx, s.g2, x)
        assert err.value.code == _lib.B200_ERR_NOT_ON_CURVE and "check %d:" % first in str(err.value), \
            (m, sorted(bad), str(err.value))

    c0 = next(c for c in range(3000, 4097) if live[c])
    c1 = next(c for c in range(2500, 4097) if live[c])
    refused({c0: pc.off_curve(g1[c0, j])}, c0)
    refused({c1: pc.plus_q(g1[c1, j], 0)}, c1)
    refused({4096: pc.plus_q(g1[4096, j] if live[4096] else pc.G1_GEN, 1)}, 4096)
    refused({64: pc.off_curve(pc.G1_GEN), c0: pc.plus_q(g1[c0, j], 1)}, 64)
    refused({c0: pc.off_curve(g1[c0, j]), c1: pc.plus_q(g1[c1, j], 0)}, min(c0, c1))
    # the context goes on checking
    assert_same(pairing_check_many(ctx, s.g2, g1), s.predicted(rows), "after the refusals", m)


# ---- the G2 generator is not hard-wired ------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def g2_pairs(srs_2_16_g2):
    """(H, tau H) of srs_2_16 and (kH, k tau H) for a seeded k"""
    h, tau_h = srs_2_16_g2
    rec = lambda p: np.frombuffer(pr.encode_g2_mont(pr.g2_mul(pr.decode_g2_mont(p.tobytes(), 0), G2_K)),
                                  dtype=np.uint64).copy()
    return (h, tau_h), (rec(h), rec(tau_h))


@pytest.fixture(scope="module")
def env_2_16(ctx, srs_2_16, g2_pairs):
    """the proofs and link proofs of `test_gpu_batch_verify.py`'s shapes, made on srs_2_16"""
    e = Env()
    e.ctx = ctx
    e.srs = rb.parse_ptau_file(ctx, srs_2_16, count=512).powers_of_g
    e.h, e.tau_h = g2_pairs[0]
    e.keys, e.proofs = [], []
    for ki, (log_n, ni, seed) in enumerate(SPECS):
        circ = synth.synth_circuit(log_n, num_inputs=ni, seed=seed, check=True,
                                   link=(LAYOUT.alignment, LAYOUT.offset, LINK_VALS))
        pk = PlonkKzgSnark.preprocess(ctx, e.srs, log_n, ni, circ.selectors, circ.perm, circ.k)
        e.keys.append((pk, VerifyingKey.from_proving_key(pk, e.h, e.tau_h)))
        for j in range(2):
            proof, hint = PlonkKzgSnark.prove_with_link_hint(ctx, pk, circ.wires, circ.pub_inputs,
                                                             synth.splitmix_blinders(2000 * ki + j))
            e.proofs.append((ki, circ.pub_inputs, proof, hint))
    e.links = []
    for a, b in ((0, 2), (2, 4), (1, 5), (4, 3)):
        lp, _ = link_proofs(ctx, e.srs, e.proofs[a][3], e.proofs[b][3], LAYOUT)
        e.links.append((e.proofs[a][3].linking_wire_comm, e.proofs[b][3].linking_wire_comm, lp, LAYOUT))
    yield e
    for pk, _ in e.keys:
        pk.free()
    e.srs.free()


def _under(items, pair):
    """the items with their verifying keys carrying the G2 pair `pair`"""
    keys = {}
    out = []
    for vk, pi, p in items:
        if id(vk) not in keys:
            keys[id(vk)] = VerifyingKey(vk.log_n, vk.num_inputs, vk.k, vk.selector_comms, vk.sigma_comms, *pair)
        out.append((keys[id(vk)], pi, p))
    return out


def _verdicts(e, items, links, pair):
    """(verify_each, batch_verify's verdicts, batch_verify's all-ok) under `pair`"""
    its = _under(items, pair)
    args = ([i[0] for i in its], [i[1] for i in its], [i[2] for i in its], links)
    each = PlonkKzgSnark.verify_each(e.ctx, *args, g2=pair)
    ok, batch = PlonkKzgSnark.batch_verify(e.ctx, *args, g2=pair)
    return each, batch, ok


def test_verifiers_under_another_g2_generator(env_2_16, g2_pairs):
    """a mixed batch of device proofs and link proofs on srs_2_16, honest and with each tampering kind of
    `test_gpu_verify_each.py` first / middle / last: per-item verdicts identical under (H, tau H) and (kH, k tau H),
    equal to the single host verifiers' under both"""
    e = env_2_16
    base, other = g2_pairs
    items = proof_items(e, [2, 0, 4, 3, 6, 1, 5, 7, 3])
    runs = [("honest", items, e.links)]
    kinds = ["eval_bit", "swap_comms", "pub_input", "wrong_vk", "off_curve", "link_layout"]
    for kind in kinds:
        n = len(e.links) if kind == "link_layout" else len(items)
        for pos in (0, n // 2, n - 1):
            runs.append(("%s at %d" % (kind, pos),) + tuple(_tamper(e, kind, items, e.links, pos)))
    # every kind in one batch, beside the honest items
    mixed_items = list(items)
    for kind, pos in zip(kinds[:-1], (0, 3, 4, 7, 8)):  # the items of the 4-input shapes
        mixed_items[pos] = _tamper(e, kind, items, e.links, pos)[0][pos]
    runs.append(("mixed", mixed_items, _tamper(e, "link_layout", items, e.links, 1)[1]))
    for name, its, lks in runs:
        want = None
        for pair in (base, other):
            single = [PlonkKzgSnark.verify(vk, pi, p) for vk, pi, p in _under(its, pair)]
            single += [verify_link_proof(a, b, lp, lay, *pair) for a, b, lp, lay in lks]
            want = single if want is None else want
            assert single == want, (name, "single verifiers differ under the second pair")
            each, batch, ok = _verdicts(e, its, lks, pair)
            assert each == want and batch == want and ok == all(want), (name, pair is other, each, batch, want)
        if name == "honest":
            assert all(want)
        elif name == "mixed":
            assert want.count(False) == 6
        else:
            assert want.count(False) == 1, name


def test_srs_check_under_another_g2_generator(ctx, oracle, srs_2_16, g2_pairs):
    """b200_srs_check of srs_2_16 against (kH, k tau H): consistent, G2 subgroup flag set; one replaced power located
    by k_srs_pairs on lines prepared from kH and k tau H; the swapped pair fails every pair"""
    pts = seeded_points(srs_2_16)
    n = pts.shape[0]
    h, bh = g2_pairs[1]
    assert rb.backend.g2_in_subgroup(h) and rb.backend.g2_in_subgroup(bh)
    assert check(ctx, pts, h, bh) == rb.SrsReport(True, True, True, 0, [])
    other = oracle.srs_from_tau(oracle.int_to_limbs(py.to_mont(OTHER_TAU % R, R)), 70)
    for j, rec in ((1, g1_dbl(oracle, pts[1])), (63, g1_neg(pts[63])), (64, other[64]), (n // 2, g1_neg(pts[n // 2])),
                   (n - 1, g1_dbl(oracle, pts[n - 1]))):
        bad = pts.copy()
        bad[j] = rec
        rep = check(ctx, bad, h, bh)
        want = expected_pairs(j, n)
        assert not rep.consistent and rep.g2_subgroup and rep.n_bad == len(want) and rep.bad == want, (j, rep)
    rep = check(ctx, pts[:512], bh, h)
    assert not rep.consistent and rep.n_bad == 511 and rep.bad == list(range(8)), rep
