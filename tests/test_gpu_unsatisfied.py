"""Refusals on the device: every witness of the violation catalogue (tests/unsat_shapes.py) gets the status the oracle
returns, through every entry point that proves — b200_plonk_prove (the first, eager proof of a key and a replayed
graph), prove_witness, prove_batch and prove_witness_batch (a refused item first, in the middle, last, and every item
refused), a pool job, a bundle and a settlement.  Satisfied items of the same call equal the oracle's bytes and the
single proof's; refused batch items and settlements are zeroed; the error names WrongQuotientPolyDegree; after every
refusal the same warm context proves a control with the same bytes in 7 graph submissions.

The low-degree cases (violations that are the values on H of a polynomial of degree <= 7) pass round 3's degree check
from n = 16 on, where the quotient is interpolated from six cosets; the prover's self-check at zeta refuses them.
The oracle's rc is computed here up to 2^10; at 2^16 and 2^17 it is the catalogue's claim (the oracle's quotient is
exact; tests/test_unsat_shapes_cpu.py checks its refusals on the same builders)."""
import numpy as np
import pytest

import unsat_shapes as us
from renegade_b200 import _lib, synth
from renegade_b200.backend import GroupLayout, PlonkKzgSnark, ProverPool

pytestmark = pytest.mark.gpu

TAU = 0x1D2C3B4A59687706F5E4D3C2B1A09F8E7D6C5B4A39281706F5E4D3C2B1A0987
UNSAT = -7
ORACLE_MAX_LOG_N = 10


class Keyed:
    """A case's SRS, table key and (where the case has a witness vector) wiring key on one context."""

    def __init__(self, ctx, oracle, pyoracle, case):
        self.case = case
        self.sel, self.wires, self.pub, self.perm, self.k, self.bl = case.tables()
        self.tau = oracle.int_to_limbs(pyoracle.to_mont(TAU % us.R, us.R))
        self.srs = oracle.srs_from_tau(self.tau, case.n + 3)
        self.bases = ctx.load_bases(self.srs)
        self.pk = PlonkKzgSnark.preprocess(ctx, self.bases, case.log_n, case.num_inputs, self.sel, self.perm, self.k)
        self.wpk = None
        if case.witness is not None:
            self.wpk = PlonkKzgSnark.preprocess_wiring(ctx, self.bases, case.log_n, case.num_inputs, self.sel,
                                                       case.wire_vars, len(case.witness), self.k)
        good_wires, good_pub = case.good
        self.good_wires = np.stack([synth.to_mont_array(c) for c in good_wires])
        self.good_pub = synth.to_mont_array(good_pub).reshape(-1, 4)

    def oracle_rc(self, oracle, wires=None, pub=None):
        """(rc, proof bytes) of the oracle, or the catalogue's claim above ORACLE_MAX_LOG_N"""
        c = self.case
        if c.log_n > ORACLE_MAX_LOG_N:
            return c.expect, None
        opk = oracle.plonk_preprocess(c.log_n, self.sel, self.perm, self.k, self.srs)
        rc, proof, _, _ = oracle.plonk_prove(c.log_n, c.num_inputs, self.k, opk, self.wires if wires is None else wires,
                                             self.pub if pub is None else pub, self.bl, self.srs)
        return rc, bytes(proof)

    def free(self):
        for k in (self.pk, self.wpk, self.bases):
            if k is not None:
                k.free()


def prove(ctx, pk, wires, pub, bl):
    """(status, proof bytes)"""
    try:
        return 0, bytes(PlonkKzgSnark.prove_with_link_hint(ctx, pk, wires, pub, bl)[0])
    except _lib.B200Error as e:
        assert e.code == UNSAT and "WrongQuotientPolyDegree" in str(e), e
        return UNSAT, None


def _status(rc):
    return UNSAT if rc == us.UNSAT else rc


def _cases():
    out = us.catalogue(ORACLE_MAX_LOG_N)
    out += [us.low_degree(16, p) for p in us.LOW_DEGREE] + [us.low_degree(17, "roots7")]
    return out


CASES = _cases()


@pytest.mark.parametrize("case", CASES, ids=[c.name for c in CASES])
def test_status_is_the_oracles_and_the_context_keeps_proving(ctx, oracle, pyoracle, case):
    ctx.use_graphs(True)
    kd = Keyed(ctx, oracle, pyoracle, case)
    try:
        want_rc, want_bytes = kd.oracle_rc(oracle)
        assert want_rc == case.expect
        # the first, eager proof of the key
        st, got = prove(ctx, kd.pk, kd.wires, kd.pub, kd.bl)
        assert st == _status(want_rc), (case.name, case.kind, "round 3 misses" if us.degree_check_misses(
            case.log_n, case.deg_r if case.deg_r is not None else case.n) else "")
        if st == 0 and want_bytes is not None:
            assert got == want_bytes
        # a control of the same key, then the case again, from replayed graphs, then the control in 7 submissions
        ctl_bl = synth.splitmix_blinders(case.log_n)
        st_c, ctl = prove(ctx, kd.pk, kd.good_wires, kd.good_pub, ctl_bl)
        assert st_c == 0
        if case.log_n <= ORACLE_MAX_LOG_N:
            opk = oracle.plonk_preprocess(case.log_n, kd.sel, kd.perm, kd.k, kd.srs)
            rc, op, _, _ = oracle.plonk_prove(case.log_n, case.num_inputs, kd.k, opk, kd.good_wires, kd.good_pub, ctl_bl, kd.srs)
            assert rc == 0 and bytes(op) == ctl
        assert prove(ctx, kd.pk, kd.wires, kd.pub, kd.bl) == (st, got)
        g0 = ctx.graph_launches()
        assert prove(ctx, kd.pk, kd.good_wires, kd.good_pub, ctl_bl) == (0, ctl)
        assert ctx.graph_launches() - g0 == 7
        # the witness-vector path of the same case
        if kd.wpk is not None:
            w = case.witness_mont()
            try:
                proof = PlonkKzgSnark.prove_witness(ctx, kd.wpk, w, kd.bl)[0]
                assert st == 0 and bytes(proof) == got
            except _lib.B200Error as e:
                assert e.code == UNSAT == st and "WrongQuotientPolyDegree" in str(e)
    finally:
        kd.free()


BATCH_CASES = ["low_degree_5_const", "low_degree_10_roots7", "single_row_5_16"]


def _by_name(name):
    return next(c for c in CASES if c.name == name)


@pytest.mark.parametrize("name", BATCH_CASES)
def test_batches_refuse_each_bad_item_and_prove_the_others(ctx, oracle, pyoracle, name):
    case = _by_name(name)
    kd = Keyed(ctx, oracle, pyoracle, case)
    try:
        bls = [synth.splitmix_blinders(900 + i) for i in range(5)]
        good = [prove(ctx, kd.pk, kd.good_wires, kd.good_pub, b)[1] for b in bls]
        zero = bytes(len(good[0]))
        w_good, w_bad = case.good_witness_mont(), case.witness_mont()
        for layout in ("GBGGB", "BGGGG", "GGGGB", "GGBGG", "BBB"):
            bad = [ch == "B" for ch in layout]
            k = len(layout)
            proofs, _, st = PlonkKzgSnark.prove_batch(ctx, kd.pk, [kd.wires if b else kd.good_wires for b in bad],
                                                      [kd.pub if b else kd.good_pub for b in bad], bls[:k])
            assert st == [UNSAT if b else 0 for b in bad], layout
            for i in range(k):
                assert bytes(proofs[i]) == (zero if bad[i] else good[i]), (layout, i)
            proofs, _, st2, _ = PlonkKzgSnark.prove_witness_batch(ctx, kd.wpk, [w_bad if b else w_good for b in bad],
                                                                  bls[:k])
            assert st2 == st, layout
            for i in range(k):
                assert bytes(proofs[i]) == (zero if bad[i] else good[i]), (layout, i)
    finally:
        kd.free()


def test_pool_bundle_and_settlement_refuse_a_low_degree_violation(oracle, pyoracle):
    case = us.low_degree(5, "const")
    pool = ProverPool(device=0, workers=2)
    try:
        pc = pool.context(0)
        kp = Keyed(pc, oracle, pyoracle, case)
        bl = synth.splitmix_blinders(77)
        want = prove(pc, kp.pk, kp.good_wires, kp.good_pub, bl)[1]
        bad = np.ascontiguousarray(kp.wires)
        good = np.ascontiguousarray(kp.good_wires)
        with pytest.raises(_lib.B200Error) as err:  # one pool job
            pool.wait(pool.submit_prove(kp.pk, bad.ctypes.data, kp.pub, bl, keep=bad))
        assert err.value.code == UNSAT and "WrongQuotientPolyDegree" in str(err.value)
        # a bundle: the refused proof fails the ticket and no link is made for it
        layout = GroupLayout(alignment=case.log_n, offset=1, size=2)
        t = pool.submit_bundle(kp.bases, [(kp.pk, good.ctypes.data, kp.good_pub, bl), (kp.pk, bad.ctypes.data, kp.pub, bl)],
                               [(0, 1, layout)])
        with pytest.raises(_lib.B200Error) as err:
            pool.wait(t)
        assert err.value.code == UNSAT
        assert pool.stats()["queued"] == 0
        ok = pool.wait(pool.submit_prove(kp.pk, good.ctypes.data, kp.good_pub, bl, keep=good))
        assert bytes(ok) == want
        # a settlement: every status refused, the proof and every link proof zeroed
        _, hint = PlonkKzgSnark.prove_with_link_hint(pc, kp.pk, kp.good_wires, kp.good_pub, bl)
        proof, lps, st = PlonkKzgSnark.prove_settlement(pc, kp.bases, kp.pk, kp.wires, kp.pub, bl, [(hint, layout)])
        assert st == [UNSAT, UNSAT]
        assert not any(bytes(proof)) and not any(bytes(lps[0]))
        proof, lps, st = PlonkKzgSnark.prove_settlement(pc, kp.bases, kp.pk, kp.good_wires, kp.good_pub, bl,
                                                        [(hint, layout)])
        assert st == [0, 0] and bytes(proof) == want
        kp.free()
    finally:
        pool.close()
