"""The collaborative prover's shapes without a GPU (tests/collab_shapes.py on `HostBackend`): the boundary claims the
device tests stand on, read from the sources; round 3 of the joint prover restated with Python integers — with its 8
cosets a violation r = X^d leaves a non-zero quotient coefficient in [5n + 8, 8n) for every d < n, n = 4 … 2^10, so
the opened tail refuses every unsatisfied witness; the share patterns; byte parity with the oracle for 1, 2, 3 parties,
every share pattern and the public-input edges at small n; every case of the violation catalogue up to 2^5 refused or
proved as the oracle does; and what the parties open."""
import numpy as np
import pytest

import collab_shapes as cs
import unsat_shapes as us
from host_backend import HostBackend
from renegade_b200 import synth
from renegade_b200 import collaborative as co
from test_unsat_shapes_cpu import G, round3_quotient

R = cs.R
TAU = 0x1D2C3B4A59687706F5E4D3C2B1A09F8E7D6C5B4A39281706F5E4D3C2B1A0987
SMALL_CASES = [c for c in us.catalogue(10) if c.log_n <= 5]


# ---- the claims the device sweep relies on ------------------------------------------------------------------------------
def test_boundaries_from_the_sources():
    sweep = list(range(2, 15)) + [16]                      # test_gpu_collaborative_shapes.py's domains
    assert cs.JOINT_COSETS == 8
    # the single prover's coset switch lies inside the sweep, with domains on both sides
    assert min(sweep) < cs.COSET_SWITCH <= max(sweep) and cs.NC_LARGE < cs.JOINT_COSETS == cs.NC_SMALL
    # m = 8n below, exactly at and above one block of the batch inversion
    ms = {cs.JOINT_COSETS << s for s in sweep}
    assert min(ms) < cs.INV_BLOCK and cs.INV_BLOCK in ms and 2 * cs.INV_BLOCK in ms
    assert cs.JOINT_COSETS << 9 == cs.INV_BLOCK
    # the wire polynomials (n + 2) and z (n + 3) reach every level count of the Horner scans, and the first domain of
    # each new level count (n = CH^k) is in the sweep
    for extra in (2, 3):
        lv = [cs.levels((1 << s) + extra) for s in sweep]
        assert sorted(set(lv)) == list(range(1, max(lv) + 1))
        for k in range(1, max(lv)):
            first = next(s for s in sweep if cs.levels((1 << s) + extra) == k + 1)
            assert 1 << first == cs.CH ** k and cs.levels((1 << (first - 1)) + extra) == k


# ---- round 3 with 8 cosets -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("log_n", [2, 3])
def test_quotient_blocks_are_the_interpolation(log_n):
    """The closed form of `quotient_blocks` = the full interpolation of test_unsat_shapes_cpu.py (per-coset inverse
    transforms, Vandermonde un-mixing) for every monomial, with 8 and 6 cosets."""
    n = 1 << log_n
    for nc in (cs.JOINT_COSETS, cs.NC_LARGE):
        a = cs.quotient_blocks(log_n, nc, G)
        for d in range(n):
            q = round3_quotient(log_n, nc, [0] * d + [1])
            assert q == [a[i // n] if i % n == d else 0 for i in range(nc * n)], (nc, d)


@pytest.mark.parametrize("log_n", range(2, 11))
def test_eight_cosets_refuse_every_violation(log_n):
    n = 1 << log_n
    for d in range(n):
        assert cs.round3_refuses_monomial(log_n, cs.JOINT_COSETS, d), d
    # the same restatement gives the single prover's 6-coset rule: X^d with d <= 7 is missed from n = 16 on
    if log_n >= 4:
        for d in range(n):
            assert cs.round3_refuses_monomial(log_n, cs.NC_LARGE, d) == (d > 7), d


# ---- share patterns --------------------------------------------------------------------------------------------------------
def test_share_patterns_are_what_they_claim():
    table = cs.mont([0, 1, R - 1, 5, 2 ** 200 + 3, 7])
    t = cs.ints(table)
    for pattern, counts in cs.PATTERNS.items():
        for p in counts:
            sh = cs.share(table, p, pattern, seed=3)
            assert len(sh) == p and cs.summed(sh) == t, pattern
            vals = [cs.ints(s) for s in sh]
            if pattern == "zero_party0":
                assert vals[0] == [0] * len(t)
            if pattern == "equal":
                assert all(v == vals[0] for v in vals)
            if pattern == "minus_one":
                assert vals[0] == [R - 1] * len(t)
            if pattern == "cancel":
                assert [(a + b) % R for a, b in zip(vals[0], vals[1])] == [0] * len(t) and vals[2] == t
            if pattern in ("random", "zero_party0") and p - (pattern == "zero_party0") > 1:
                assert all(v != t for v in vals)
    # one party: share_table and the Dealer degenerate to the clear table
    assert (co.share_table(table, 1, seed=9)[0] == table).all()
    be = HostBackend(np.zeros((1, 8), dtype=np.uint64))
    d = co.Dealer(be, 1)
    a, b, c = d.triple(4)
    assert [x * y % R for x, y in zip(a[0].v, b[0].v)] == c[0].v
    bl = cs.nonzero_blinder_split(synth.splitmix_blinders(3), 3, seed=4)
    assert all(all(cs.ints(s)) for s in bl) and cs.summed(bl) == cs.ints(synth.splitmix_blinders(3))


# ---- parity on the host backend ----------------------------------------------------------------------------------------
def _tau(oracle, pyoracle):
    return oracle.int_to_limbs(pyoracle.to_mont(TAU % R, R))


def joint_parity(oracle, pyoracle, log_n, num_inputs, sel, perm, k, wires, pub, bl, wire_shares, bl_shares):
    """The opened proof = the oracle's proof of the summed witness and blinders, hint included; known-τ verified."""
    tau = _tau(oracle, pyoracle)
    srs = oracle.srs_from_tau(tau, (1 << log_n) + 3)
    opk = oracle.plonk_preprocess(log_n, sel, perm, k, srs)
    rc, oproof, _, olink = oracle.plonk_prove(log_n, num_inputs, k, opk, wires, pub, bl, srs, True)
    assert rc == 0
    be = HostBackend(srs)
    cpk = co.CollaborativeProvingKey.build(be, log_n, num_inputs, sel, perm, k)
    assert (cpk.selector_comms == opk["selector_comms"]).all() and (cpk.sigma_comms == opk["sigma_comms"]).all()
    proof, hint, fab = co.MultiproverPlonkKzgSnark.prove_with_link_hint(be, cpk, wire_shares, pub, bl_shares)
    assert bytes(proof) == bytes(oproof)
    assert (hint.linking_wire_poly == olink).all()
    assert oracle.plonk_verify_known_tau(log_n, num_inputs, k, opk, pub, oracle.PlonkProof.from_buffer_copy(bytes(proof)), tau)
    return proof, hint, fab


@pytest.mark.parametrize("log_n,parties,num_inputs,pattern", [
    (2, 1, 1, "random"), (4, 1, 3, "random"), (3, 5, 1, "random"),
    (5, 2, 0, "random"), (5, 2, 1, "random"), (5, 2, 5, "random"), (5, 2, "all", "random"),
] + [(5, p, 3, pat) for pat, counts in cs.PATTERNS.items() for p in counts])
def test_joint_proof_equals_oracle(oracle, pyoracle, log_n, parties, num_inputs, pattern):
    circ = cs.circuit(log_n, num_inputs)
    bl = synth.splitmix_blinders(500 + log_n)
    ws = cs.share(np.asarray(circ.wires, dtype=np.uint64).reshape(-1, 4), parties, pattern, seed=11)
    bs = cs.share(np.asarray(bl, dtype=np.uint64).reshape(-1, 4), parties, pattern, seed=12)
    joint_parity(oracle, pyoracle, log_n, circ.num_inputs, circ.selectors, circ.perm, circ.k, circ.wires, circ.pub_inputs,
                 bl, ws, bs)


# ---- the violation catalogue up to 2^5 --------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", SMALL_CASES, ids=[c.name for c in SMALL_CASES])
def test_catalogue_on_the_host_backend(oracle, pyoracle, case):
    srs = oracle.srs_from_tau(_tau(oracle, pyoracle), case.n + 3)
    be = HostBackend(srs)

    def prove_joint(sel, perm, k, wires, pub, ws, bs):
        cpk = co.CollaborativeProvingKey.build(be, case.log_n, case.num_inputs, sel, perm, k)
        return co.MultiproverPlonkKzgSnark.prove_with_link_hint(be, cpk, ws, pub, bs)[0]

    cs.catalogue_case(oracle, _tau(oracle, pyoracle), case, prove_joint)


# ---- what the parties open ---------------------------------------------------------------------------------------------------
def opened_vectors(monkeypatch, run):
    """Run `run()` with `collaborative.Fabric` replaced by a subclass that records every opened vector (as integers)."""
    seen = []

    class Recording(co.Fabric):
        def open(self, x):
            acc = super().open(x)
            seen.append(cs.ints(self.be.to_limbs(acc)))
            return acc

    monkeypatch.setattr(co, "Fabric", Recording)
    return run(), seen


def test_nothing_but_the_documented_openings(oracle, pyoracle, monkeypatch):
    """At 2^5 with 2 parties: no opened vector contains a wire column of the summed table or z's evaluations over H,
    except the two documented openings (`collab_shapes.check_openings`)."""
    log_n = 5
    circ = cs.circuit(log_n, 3)
    bl = synth.splitmix_blinders(77)
    ws = cs.share(np.asarray(circ.wires, dtype=np.uint64).reshape(-1, 4), 2, "random", seed=21)
    bs = cs.share(np.asarray(bl, dtype=np.uint64).reshape(-1, 4), 2, "random", seed=22)
    (proof, hint, fab), seen = cs.opened_vectors(monkeypatch, lambda: joint_parity(
        oracle, pyoracle, log_n, circ.num_inputs, circ.selectors, circ.perm, circ.k, circ.wires, circ.pub_inputs, bl, ws, bs))
    tau = _tau(oracle, pyoracle)
    srs = oracle.srs_from_tau(tau, (1 << log_n) + 3)
    opk = oracle.plonk_preprocess(log_n, circ.selectors, circ.perm, circ.k, srs)
    _, _, ch, _ = oracle.plonk_prove(log_n, circ.num_inputs, circ.k, opk, circ.wires, circ.pub_inputs, bl, srs)
    cs.check_openings(circ, hint, seen, ch, lambda v: cs.ints(oracle.ntt(cs.mont(v))))
    assert len(seen) > 10 and fab.opened_elements >= sum(len(v) for v in seen)
