"""GPU parity of the link division (`link` in plonk.cu) at the layouts where it departs from the reference's `size`
successive synthetic divisions: the device divides pointwise by Z_D on a coset of N = 2^k >= len points and tests the
quotient's degree over coefficients [q_len, N).  The inputs are built from the algebra (`link_layouts.py`, whose shapes
`test_link_layouts_cpu.py` pins): size 1, q_len 1, the whole subgroup (Z_D = X^(2^a) - 1), roots wrapping past g^0,
an alignment above log2 N, len = N, len1 < len2 and len1 > len2 at several ratios, equal polynomials (identity quotient
and opening commitments) and the largest SRS.  Each link proof and eta are byte-equal to the oracle's and accepted by the
oracle's and the product's link verifiers and by one batch verification; a difference on exactly one root is refused
and the context keeps proving; a replayed graph gives the oracle's proof for new polynomials."""
import numpy as np
import pytest

import link_layouts as ll
from renegade_b200._lib import B200Error
from renegade_b200.backend import GroupLayout, LinkingHint, PlonkKzgSnark, link_proofs, verify_link_proof

pytestmark = pytest.mark.gpu

TAU = 0x1D2C3B4A59687706F5E4D3C2B1A09F8E7D6C5B4A39281706F5E4D3C2B1A0987  # conftest's SRS_2_16_TAU: srs_2_16_g2 is its G2 pair
NAMES = [c.name for c in ll.CASES]
UNSAT = -7


@pytest.fixture(scope="module")
def env(ctx, oracle, srs_2_16_g2):
    class E:
        pass
    e = E()
    e.ctx, e.oracle = ctx, oracle
    e.tau = oracle.int_to_limbs(TAU % ll.R * ll.MONT % ll.R)
    e.srs = oracle.srs_from_tau(e.tau, (1 << 17) + 3)
    assert max(c.len for c in ll.CASES) == e.srs.shape[0] - 1
    e.bases = ctx.load_bases(e.srs)
    e.h, e.tau_h = srs_2_16_g2
    e.done = {}  # case name -> (c1, c2, link proof, layout)
    yield e
    e.bases.free()


def hint(e, vals):
    m = ll.to_mont(vals)
    xy, inf = e.ctx.msm(e.bases, m, montgomery=True)
    return LinkingHint(m, np.zeros(8, dtype=np.uint64) if inf else xy)


def layout(c):
    return GroupLayout(c.alignment, c.offset, c.size)


def prove_and_compare(e, c, a1, a2):
    """device link proof of (a1, a2) = oracle's, byte for byte; both link verifiers accept it"""
    h1, h2 = hint(e, a1), hint(e, a2)
    lp, eta = link_proofs(e.ctx, e.bases, h1, h2, layout(c))
    rc, olp, oeta = e.oracle.plonk_link(h1.linking_wire_poly, h2.linking_wire_poly, h1.linking_wire_comm,
                                        h2.linking_wire_comm, c.alignment, c.offset, c.size, e.srs)
    assert rc == 0
    assert bytes(lp) == bytes(olp)
    assert eta.tobytes() == oeta.tobytes()
    assert e.oracle.plonk_link_verify_known_tau(h1.linking_wire_comm, h2.linking_wire_comm, c.alignment, c.offset, c.size,
                                                e.oracle.LinkProof.from_buffer_copy(bytes(lp)), e.tau)
    assert verify_link_proof(h1.linking_wire_comm, h2.linking_wire_comm, lp, layout(c), e.h, e.tau_h)
    return h1, h2, lp


def proved(e, c):
    if c.name not in e.done:
        a1, a2 = ll.pair(e.oracle, c, seed=0x11 + NAMES.index(c.name))
        h1, h2, lp = prove_and_compare(e, c, a1, a2)
        e.done[c.name] = (h1.linking_wire_comm, h2.linking_wire_comm, lp, layout(c))
    return e.done[c.name]


@pytest.mark.parametrize("name", NAMES)
def test_link_layout_matches_oracle(env, name):
    c = ll.BY_NAME[name]
    assert ll.domain_n(c.len) == c.N and c.len - c.size == c.q_len  # the shape test_link_layouts_cpu.py pins
    c1, c2, lp, _ = proved(env, c)
    # equal polynomials: the zero quotient commits to the identity, encoded (as in the transcript) as 64 zero bytes
    assert (not lp.to_array()[:8].any()) == c.identical and (not lp.to_array()[8:].any()) == c.identical
    assert (c1 == c2).all() == c.identical


def test_batch_verification_of_every_layout(env):
    links = [proved(env, c) for c in ll.CASES]
    ok, verdicts = PlonkKzgSnark.batch_verify(env.ctx, [], [], [], links, g2=(env.h, env.tau_h))
    assert ok and verdicts == [True] * len(links)
    for i, c in enumerate(ll.CASES):
        # one row further: other roots — except for the whole subgroup (the same roots) and equal polynomials
        keeps = c.identical or c.size == 1 << c.alignment
        a, b, lp, lay = links[i]
        shifted = links[:i] + [(a, b, lp, GroupLayout(lay.alignment, lay.offset + 1, lay.size))] + links[i + 1:]
        ok, verdicts = PlonkKzgSnark.batch_verify(env.ctx, [], [], [], shifted, g2=(env.h, env.tau_h))
        assert ok == keeps and verdicts == [j != i or keeps for j in range(len(links))], c.name
        assert verify_link_proof(a, b, lp, shifted[i][3], env.h, env.tau_h) == keeps


@pytest.mark.parametrize("j", ["first", "middle", "last"])
def test_one_root_mismatch_is_refused(env, j):
    """a1 + c * Z_D / (X - root_j) differs from a2 on root j only ("middle" is g^8 = 1, where the roots wrap)"""
    c = ll.BY_NAME["wraps"]
    idx = {"first": 0, "middle": c.size // 2, "last": c.size - 1}[j]
    honest = proved(env, c)
    a1, a2 = ll.pair(env.oracle, c, seed=0x11 + NAMES.index(c.name))
    bad = ll.mismatch(env.oracle, c, a1, idx, 0xC0FFEE + idx)
    d = ll.poly_add(bad, a2, -1)
    rts = ll.roots(env.oracle, c)
    assert [ll.poly_eval(d, r) != 0 for r in rts] == [i == idx for i in range(c.size)]
    assert (rts[idx] == 1) == (j == "middle")
    h1, h2 = hint(env, bad), hint(env, a2)
    with pytest.raises(B200Error) as err:
        link_proofs(env.ctx, env.bases, h1, h2, layout(c))
    assert err.value.code == UNSAT
    rc, _, _ = env.oracle.plonk_link(h1.linking_wire_poly, h2.linking_wire_poly, h1.linking_wire_comm, h2.linking_wire_comm,
                                     c.alignment, c.offset, c.size, env.srs)
    assert rc == 2
    # the context still proves the honest pair
    lp, _ = link_proofs(env.ctx, env.bases, hint(env, a1), hint(env, a2), layout(c))
    assert bytes(lp) == bytes(honest[2])


def test_graph_replay_with_new_polynomials(env):
    """one layout three times (eager, captured, replayed), different polynomials each time: the oracle's proof each time"""
    c = ll.Case("replay", 6, 33, 9, 50, 45, N=64, q_len=41)
    env.ctx.use_graphs(True)
    submissions, proofs = [], set()
    for rnd in range(3):
        a1, a2 = ll.pair(env.oracle, c, seed=0x5EED + rnd)
        g0 = env.ctx.graph_launches()
        _, _, lp = prove_and_compare(env, c, a1, a2)
        submissions.append(env.ctx.graph_launches() - g0)
        proofs.add(bytes(lp))
    assert submissions == [0, 2, 2] and len(proofs) == 3
