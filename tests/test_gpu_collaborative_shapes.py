"""The collaborative prover on the device (renegade_b200/collaborative.py on `DeviceBackend`) at the shapes of
tests/collab_shapes.py.  "Parity" is: the opened proof's bytes = the device single-prover proof's = the oracle's proof
of the summed witness with the summed blinders (a mismatch names the differing proof fields); the hint's linking
polynomial and commitment = the single prover's (and the oracle's polynomial); the `CollaborativeProvingKey`
commitments = the device key's; the opened proof accepted by the oracle's known-τ verifier and by `b200_plonk_verify`.

Every domain 2^2 … 2^14 and 2^16 (across the single prover's coset switch, the batch inversion's block, every level
count of the Horner scans); 1, 3, 5 parties; no, one, five and every row public; the share patterns (party 0 all
zero, equal shares, r − 1 / t + 1, shares that cancel); every case of the violation catalogue refused or proved as
the oracle does (8 cosets: the low-degree violations the single prover only refuses at ζ are refused in round 3);
joint proofs between captured and replayed proofs of another key on one context, in both orders; the benchmark's
joint proof, also under a side stream; both multiprover statements and the private-match link proofs made from the
opened hint; and what the parties open."""
import contextlib
import functools
import random

import numpy as np
import pytest
import torch

import collab_shapes as cs
import unsat_shapes as us
from conftest import SRS_2_16_TAU
from renegade_b200 import collaborative as co
from renegade_b200 import synth
from renegade_b200.backend import B200Proof, PlonkKzgSnark, VerifyingKey

pytestmark = pytest.mark.gpu

R = cs.R
NAMES = ["wire_comm"] * 40 + ["z_comm"] * 8 + ["quot_comm"] * 40 + ["opening"] * 8 + ["shifted"] * 8 + \
        ["wire_eval"] * 20 + ["sigma_eval"] * 16 + ["z_next"] * 4
SWEEP = list(range(2, 15)) + [16]
_ORACLE = {}


@pytest.fixture(scope="module")
def tau(oracle, pyoracle):
    """τ of the srs_2_16 fixture: every SRS here is its first n + 3 powers."""
    return oracle.int_to_limbs(pyoracle.to_mont(SRS_2_16_TAU % R, R))


def assert_same_proof(ours, theirs, what):
    a = ours.to_array()
    b = B200Proof.from_buffer_copy(bytes(theirs)).to_array()
    diff = sorted({NAMES[i] for i in range(len(NAMES)) if a[i] != b[i]})
    assert not diff, (what, diff)


@functools.lru_cache(maxsize=None)
def circuit(log_n, num_inputs):
    return cs.circuit(log_n, num_inputs)


def oracle_key(oracle, tau, circ):
    """(srs, oracle key) of a circuit of `circuit()`, cached."""
    key = ("pk", circ.log_n, circ.num_inputs, id(circ))
    if key not in _ORACLE:
        srs = oracle.srs_from_tau(tau, circ.n + 3)
        _ORACLE[key] = (srs, oracle.plonk_preprocess(circ.log_n, circ.selectors, circ.perm, circ.k, srs))
    return _ORACLE[key]


def oracle_proof(oracle, tau, circ, bl, key):
    """(srs, oracle key, oracle proof, oracle linking polynomial), cached by `key` across the tests of this file."""
    if key not in _ORACLE:
        srs, opk = oracle_key(oracle, tau, circ)
        rc, proof, _, link = oracle.plonk_prove(circ.log_n, circ.num_inputs, circ.k, opk, circ.wires, circ.pub_inputs, bl,
                                                srs, True)
        assert rc == 0
        _ORACLE[key] = (srs, opk, proof, link)
    return _ORACLE[key]


def joint(ctx, bases, circ, wire_shares, bl_shares):
    be = co.DeviceBackend(ctx, bases)
    cpk = co.CollaborativeProvingKey.build(be, circ.log_n, circ.num_inputs, circ.selectors, circ.perm, circ.k)
    proof, hint, fab = co.MultiproverPlonkKzgSnark.prove_with_link_hint(be, cpk, wire_shares, circ.pub_inputs, bl_shares)
    return cpk, proof, hint, fab


def parity(ctx, oracle, tau, g2, circ, parties, pattern="random", bl_seed=90, key=None):
    bl = synth.splitmix_blinders(bl_seed + circ.log_n)
    ws = cs.share(np.asarray(circ.wires, dtype=np.uint64).reshape(-1, 4), parties, pattern, seed=17)
    bs = cs.share(np.asarray(bl, dtype=np.uint64).reshape(-1, 4), parties, pattern, seed=18)
    assert cs.summed(ws) == cs.ints(circ.wires) and cs.summed(bs) == cs.ints(bl)
    srs, opk, oproof, olink = oracle_proof(oracle, tau, circ, bl, key or (circ.log_n, circ.num_inputs, bl_seed))
    bases = ctx.load_bases(srs)
    pk = None
    try:
        pk = PlonkKzgSnark.preprocess(ctx, bases, circ.log_n, circ.num_inputs, circ.selectors, circ.perm, circ.k)
        single, shint = PlonkKzgSnark.prove_with_link_hint(ctx, pk, circ.wires, circ.pub_inputs, bl)
        cpk, proof, hint, fab = joint(ctx, bases, circ, ws, bs)
        assert_same_proof(single, oproof, "single prover vs oracle")
        assert_same_proof(proof, oproof, f"joint ({parties} parties, {pattern}) vs oracle")
        assert (cpk.selector_comms == pk.selector_comms).all() and (cpk.sigma_comms == pk.sigma_comms).all()
        assert (hint.linking_wire_poly == shint.linking_wire_poly).all() and (hint.linking_wire_poly == olink).all()
        assert (hint.linking_wire_comm == shint.linking_wire_comm).all()
        assert oracle.plonk_verify_known_tau(circ.log_n, circ.num_inputs, circ.k, opk, circ.pub_inputs,
                                             oracle.PlonkProof.from_buffer_copy(bytes(proof)), tau)
        assert PlonkKzgSnark.verify(VerifyingKey.from_proving_key(pk, *g2), circ.pub_inputs, proof)
        return fab
    finally:
        if pk is not None:
            pk.free()
        bases.free()


# ---- 1. every domain -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("log_n", SWEEP)
def test_every_domain(ctx, oracle, tau, srs_2_16_g2, log_n):
    circ = circuit(log_n, 5)
    if log_n == 16:
        # z has n + 3 coefficients: its commitment takes every power of an SRS made like srs_2_16
        assert oracle_proof(oracle, tau, circ, synth.splitmix_blinders(90 + log_n), (log_n, 5, 90))[0].shape[0] == circ.n + 3
    fab = parity(ctx, oracle, tau, srs_2_16_g2, circ, 2)
    assert fab.multiplications >= 26 * cs.JOINT_COSETS * circ.n


# ---- 2. party counts and public inputs -----------------------------------------------------------------------------------------
@pytest.mark.parametrize("log_n,parties", [(s, p) for s in (2, 4, 9, 10, 12) for p in (1, 3, 5)])
def test_party_counts(ctx, oracle, tau, srs_2_16_g2, log_n, parties):
    parity(ctx, oracle, tau, srs_2_16_g2, circuit(log_n, 5), parties)


@pytest.mark.parametrize("log_n,num_inputs", [(s, ni) for s in (5, 10) for ni in (0, 1, 5, "all")])
def test_public_inputs(ctx, oracle, tau, srs_2_16_g2, log_n, num_inputs):
    circ = circuit(log_n, num_inputs)
    assert circ.num_inputs == (circ.n if num_inputs == "all" else num_inputs)
    parity(ctx, oracle, tau, srs_2_16_g2, circ, 2, key=(log_n, num_inputs, 90))


# ---- 3. share patterns -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("log_n,parties,pattern",
                         [(s, p, pat) for s in (5, 12) for pat, counts in cs.PATTERNS.items() for p in counts])
def test_share_patterns(ctx, oracle, tau, srs_2_16_g2, log_n, parties, pattern):
    parity(ctx, oracle, tau, srs_2_16_g2, circuit(log_n, 5), parties, pattern)


# ---- 4. the refusal catalogue ------------------------------------------------------------------------------------------------------
CASES = us.catalogue(10) + [us.low_degree(16, p) for p in us.LOW_DEGREE]


@pytest.mark.parametrize("case", CASES, ids=[c.name for c in CASES])
def test_catalogue(ctx, oracle, tau, case):
    """Every case with 2 parties: the verdict the oracle gives (8 cosets refuse the low-degree violations in round 3,
    at every n), each refusal followed by the case's satisfying control = oracle bytes."""
    bases = ctx.load_bases(oracle.srs_from_tau(tau, case.n + 3))
    be = co.DeviceBackend(ctx, bases)

    def prove_joint(sel, perm, k, wires, pub, ws, bs):
        cpk = co.CollaborativeProvingKey.build(be, case.log_n, case.num_inputs, sel, perm, k)
        return co.MultiproverPlonkKzgSnark.prove_with_link_hint(be, cpk, ws, pub, bs)[0]

    try:
        cs.catalogue_case(oracle, tau, case, prove_joint)
    finally:
        bases.free()


# ---- 5. one context, two provers -----------------------------------------------------------------------------------------------------
def _replays(ctx, pk, circ, oracle, tau, bl_seeds, what):
    for s in bl_seeds:
        bl = synth.splitmix_blinders(s)
        proof, _ = PlonkKzgSnark.prove_with_link_hint(ctx, pk, circ.wires, circ.pub_inputs, bl)
        assert_same_proof(proof, oracle_proof(oracle, tau, circ, bl, (circ.log_n, 5, "bl", s))[2], (what, s))


@pytest.mark.parametrize("key_log_n,joint_log_n", [(8, 16), (16, 10)])
def test_joint_between_replays(oracle, tau, key_log_n, joint_log_n):
    """A key proved eagerly, then captured, then replayed; a joint proof on the same context; the key replayed again —
    every proof = oracle bytes.  Small key first: the joint call grows plonk_ws, the NTT scratch and the MSM scratch
    under the key's captured graphs (restated from plonk.cu's reserve sizes).  Large key first: the joint call works
    in the buffers the captured graphs point at."""
    import renegade_b200 as rb
    if key_log_n < joint_log_n:
        assert cs.joint_ws_elems(joint_log_n) > cs.prover_ws_elems(key_log_n)
        assert cs.joint_inverse_elems(joint_log_n) > cs.prover_ntt_scratch_elems(key_log_n)
        assert (1 << joint_log_n) + 3 > (1 << key_log_n) + 3  # the MSM scratch grows with the number of points
    else:
        assert cs.joint_ws_elems(joint_log_n) <= cs.prover_ws_elems(key_log_n)
        assert cs.joint_inverse_elems(joint_log_n) <= cs.prover_ntt_scratch_elems(key_log_n)
    kc, jc = circuit(key_log_n, 5), circuit(joint_log_n, 5)
    ctx = rb.Context(0)
    kb = jb = pk = None
    try:
        kb = ctx.load_bases(oracle.srs_from_tau(tau, kc.n + 3))
        pk = PlonkKzgSnark.preprocess(ctx, kb, key_log_n, kc.num_inputs, kc.selectors, kc.perm, kc.k)
        _replays(ctx, pk, kc, oracle, tau, (1, 2, 1), "eager, captured, replayed")
        bl = synth.splitmix_blinders(90 + joint_log_n)
        srs, _, oproof, _ = oracle_proof(oracle, tau, jc, bl, (joint_log_n, 5, 90))
        jb = ctx.load_bases(srs)
        ws = cs.share(np.asarray(jc.wires, dtype=np.uint64).reshape(-1, 4), 2, "random", seed=17)
        bs = cs.share(np.asarray(bl, dtype=np.uint64).reshape(-1, 4), 2, "random", seed=18)
        assert_same_proof(joint(ctx, jb, jc, ws, bs)[1], oproof, "joint proof between replays")
        _replays(ctx, pk, kc, oracle, tau, (2, 1), "after the joint proof")
    finally:
        if pk is not None:
            pk.free()
        for b in (kb, jb):
            if b is not None:
                b.free()
        ctx.close()


# ---- 6. the benchmark's joint proof ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("side_stream", [False, True])
def test_benchmark_joint_proof(ctx, oracle, side_stream):
    """`bench.py`'s collaborative_leg rebuilt: the 2^12 private settlement (seed 61), known-discrete-log bases made on
    the device and loaded with window_bits=1, 2 parties, shares seeded 1 and 2, splitmix_blinders(4242); a warm-up and
    three proofs, each = the single-prover proof = the oracle's.  With side_stream, all of it under an active
    torch.cuda.stream(side): `DeviceBackend._sync` waits for torch's current stream only."""
    from host_circuits import private_settlement as ps
    seed_srs, n_srs = 0x7A0, (1 << 14) + 3  # bench.py's SEED_SRS and SRS length
    parties, statement = ps.create_witness_statement(seed=61)
    circ = ps.IntentAndBalancePrivateSettlementCircuit.build(parties, statement).finalize_for_arithmetization()
    assert circ.log_n == 12
    bl = synth.splitmix_blinders(4242)
    srs = oracle.known_dlog_bases(seed_srs, circ.n + 3)
    opk = oracle.plonk_preprocess(circ.log_n, circ.selectors, circ.perm, circ.k, srs)
    rc, oproof, _, _ = oracle.plonk_prove(circ.log_n, circ.num_inputs, circ.k, opk, circ.wires, circ.pub_inputs, bl, srs)
    assert rc == 0
    d_srs = torch.empty((n_srs, 8), dtype=torch.int64, device="cuda")
    torch.cuda.synchronize()
    ctx.known_dlog_bases_device(seed_srs, n_srs, d_srs.data_ptr())
    bases = ctx.load_bases_device(d_srs.data_ptr(), circ.n + 3, window_bits=1)
    side = torch.cuda.Stream()
    try:
        with torch.cuda.stream(side) if side_stream else contextlib.nullcontext():
            be = co.DeviceBackend(ctx, bases)
            cpk = co.CollaborativeProvingKey.build(be, circ.log_n, circ.num_inputs, circ.selectors, circ.perm, circ.k)
            shares = co.share_table(np.asarray(circ.wires, dtype=np.uint64).reshape(-1, 4), 2, seed=1)
            bsh = co.share_table(np.asarray(bl, dtype=np.uint64).reshape(-1, 4), 2, seed=2)
            proofs = [co.MultiproverPlonkKzgSnark.prove_with_link_hint(be, cpk, shares, circ.pub_inputs, bsh)[0]
                      for _ in range(4)]
        pk = PlonkKzgSnark.preprocess(ctx, bases, circ.log_n, circ.num_inputs, circ.selectors, circ.perm, circ.k)
        single, _ = PlonkKzgSnark.prove_with_link_hint(ctx, pk, circ.wires, circ.pub_inputs, bl)
        pk.free()
        assert_same_proof(single, oproof, "single prover vs oracle")
        for i, p in enumerate(proofs):
            assert_same_proof(p, oproof, ("joint proof", i, "side stream" if side_stream else "default stream"))
    finally:
        bases.free()
        del d_srs


# ---- 7. the statement surface ------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def system_srs(ctx, srs_2_16, srs_2_16_g2):
    import renegade_b200 as rb
    from renegade_b200 import circuit_types as ct
    params = rb.parse_ptau_file(ctx, srs_2_16, count=(1 << 16) + 3)
    ct.set_system_srs(ctx, params.powers_of_g, *srs_2_16_g2)
    yield params.powers_of_g
    ct.clear_key_cache()


def test_valid_balance_create_multiprover(system_srs):
    from host_circuits import statements as st
    from host_circuits import valid_balance_create as vbc
    from renegade_b200 import circuit_types as ct
    w, s = vbc.create_witness_statement(7)
    C = st.ValidBalanceCreateMultiprover
    circ, shares = C.share_witness_table(w, s, 2, seed=5)
    bl = ct.draw_blinders(random.Random(9))
    proof, hint = ct.multiprover_prove_with_hint(C, circ, shares, co.share_table(bl, 2, seed=6))
    single, shint = ct.singleprover_prove_with_hint(C.BaseCircuit, w, s, rng=random.Random(9))
    assert_same_proof(proof, single, "VALID BALANCE CREATE, 2 parties")
    assert (hint.linking_wire_poly == shint.linking_wire_poly).all()
    ct.verify_singleprover_proof(C.BaseCircuit, s, proof)
    ct.multiprover_prove_and_verify(C, w, s, parties=2, rng=random.Random(3))


def test_private_settlement_three_parties_and_its_links(ctx, system_srs, srs_2_16_g2):
    """The settlement proved by 3 parties opens to the single-prover proof; the link proofs from the parties' validity
    hints to the OPENED settlement hint = those to the single-prover hint, and the link verifier accepts them."""
    from host_circuits import intent_and_balance_validity as val
    from host_circuits import output_balance_validity as obv
    from host_circuits import private_settlement as ps
    from host_circuits import statements as st
    from renegade_b200 import circuit_types as ct
    from renegade_b200.backend import GroupLayout, link_proofs, verify_link_proof
    parties, _ = ps.create_witness_statement(seed=61)
    validity = [val.create_witness_statement(seed=70 + i, intent=parties[i].intent, balance=parties[i].input_balance)
                for i in (0, 1)]
    out_validity = [obv.create_witness_statement(80 + i, parties[i].output_balance) for i in (0, 1)]
    parties, statement = ps.create_witness_statement(
        seed=61, linked=[(validity[i][0].new_amount_public_share, validity[i][0].post_match_balance_shares,
                          out_validity[i][0].post_match_balance_shares) for i in (0, 1)])
    C = st.IntentAndBalancePrivateSettlementMultiprover
    S = C.BaseCircuit
    circ, shares = C.share_witness_table(parties, statement, 3, seed=5)
    bl = ct.draw_blinders(random.Random(9))
    proof, hint = ct.multiprover_prove_with_hint(C, circ, shares, co.share_table(bl, 3, seed=6))
    single, shint = ct.singleprover_prove_with_hint(S, parties, statement, rng=random.Random(9))
    assert_same_proof(proof, single, "private settlement, 3 parties")
    assert (hint.linking_wire_poly == shint.linking_wire_poly).all()
    assert (hint.linking_wire_comm == shint.linking_wire_comm).all()
    ct.verify_singleprover_proof(S, statement, proof)
    layouts = S.get_circuit_layout()
    h, tau_h = srs_2_16_g2
    for i in (0, 1):
        for V, (w, s_), gid in ((st.IntentAndBalanceValidityCircuit, validity[i], ps.PARTY_LINKS[i]),
                                (st.OutputBalanceValidityCircuit, out_validity[i], ps.OUTPUT_LINKS[i])):
            _, vhint = ct.singleprover_prove_with_hint(V, w, s_)
            lay = GroupLayout(layouts[gid].alignment, layouts[gid].offset, layouts[gid].size)
            lp, eta = link_proofs(ctx, system_srs, vhint, hint, lay)
            lp_single, eta_single = link_proofs(ctx, system_srs, vhint, shint, lay)
            assert bytes(lp) == bytes(lp_single) and np.array_equal(np.asarray(eta), np.asarray(eta_single)), gid
            assert verify_link_proof(vhint.linking_wire_comm, hint.linking_wire_comm, lp, lay, h, tau_h), gid


# ---- 8. what is opened -------------------------------------------------------------------------------------------------------------------
def test_nothing_but_the_documented_openings(ctx, oracle, tau, monkeypatch):
    """At 2^5 with 2 parties no opened vector contains a wire column of the summed table or z's evaluations over H.
    Two openings are documented exceptions: round 3's tail (its top coefficient, then zeros) and the hint's `link_poly`,
    the blinded wire-0 polynomial, opened whole.  That second one is a design finding: folded mod X^n − 1 it IS wire 0
    on H (asserted below), whereas the reference hands back a shared `MpcProofLinkingHint`
    (circuits-core/src/lib.rs:153-160) and never opens it."""
    log_n = 5
    circ = circuit(log_n, 3)
    bl = synth.splitmix_blinders(77)
    ws = cs.share(np.asarray(circ.wires, dtype=np.uint64).reshape(-1, 4), 2, "random", seed=21)
    bs = cs.share(np.asarray(bl, dtype=np.uint64).reshape(-1, 4), 2, "random", seed=22)
    srs, opk, oproof, _ = oracle_proof(oracle, tau, circ, bl, (log_n, 3, "openings"))
    _, _, ch, _ = oracle.plonk_prove(log_n, circ.num_inputs, circ.k, opk, circ.wires, circ.pub_inputs, bl, srs)
    bases = ctx.load_bases(srs)
    try:
        (_, proof, hint, fab), seen = cs.opened_vectors(monkeypatch, lambda: joint(ctx, bases, circ, ws, bs))
    finally:
        bases.free()
    assert_same_proof(proof, oproof, "joint proof with a recording fabric")
    cs.check_openings(circ, hint, seen, ch, lambda v: cs.ints(oracle.ntt(cs.mont(v))))
    assert len(seen) > 10 and fab.opened_elements >= sum(len(v) for v in seen)
