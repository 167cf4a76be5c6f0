"""Batch verification on the device (`b200_plonk_batch_verify`, `PlonkKzgSnark.batch_verify`): many proofs and link
proofs checked with ONE pairing must give, item by item, the answers of the single host verifiers.  Proofs come from
the device prover on the reference's SRS head (its first 512 G1 powers and its G2 pair)."""
import random

import numpy as np
import pytest

import renegade_b200 as rb
from renegade_b200 import synth
from renegade_b200.backend import (B200LinkProof, B200Proof, GroupLayout, PlonkKzgSnark, VerifyingKey, link_proofs,
                                   verify_link_proof)

pytestmark = pytest.mark.gpu

LAYOUT = GroupLayout(alignment=5, offset=20, size=6)
LINK_VALS = [(0x5EED + 77 * i) ** 3 % synth.R for i in range(LAYOUT.size)]
# (log_n, num_inputs, circuit seed): three shapes, and a second circuit of the second shape (the "wrong key")
SPECS = [(6, 0, 1), (7, 4, 2), (8, 120, 3), (7, 4, 9)]


class Env:
    pass


@pytest.fixture(scope="module")
def env(ctx, srs_head, g2_raw):
    e = Env()
    e.ctx = ctx
    e.srs = rb.parse_ptau_file(ctx, srs_head, count=512).powers_of_g
    e.h, e.tau_h = g2_raw
    e.keys, e.proofs = [], []  # proofs: (key index, pub_inputs, proof, hint)
    for ki, (log_n, ni, seed) in enumerate(SPECS):
        circ = synth.synth_circuit(log_n, num_inputs=ni, seed=seed, check=True,
                                   link=(LAYOUT.alignment, LAYOUT.offset, LINK_VALS))
        pk = PlonkKzgSnark.preprocess(ctx, e.srs, log_n, ni, circ.selectors, circ.perm, circ.k)
        e.keys.append((pk, VerifyingKey.from_proving_key(pk, e.h, e.tau_h)))
        for b in range(2):
            proof, hint = PlonkKzgSnark.prove_with_link_hint(ctx, pk, circ.wires, circ.pub_inputs,
                                                             synth.splitmix_blinders(1000 * ki + b))
            e.proofs.append((ki, circ.pub_inputs, proof, hint))
    # link proofs between proofs of different keys
    e.links = []
    for a, b in ((0, 2), (2, 4), (1, 5), (4, 3)):
        lp, _ = link_proofs(ctx, e.srs, e.proofs[a][3], e.proofs[b][3], LAYOUT)
        e.links.append((e.proofs[a][3].linking_wire_comm, e.proofs[b][3].linking_wire_comm, lp, LAYOUT))
    return e


def single_verdicts(e, items, links):
    out = [PlonkKzgSnark.verify(vk, pi, p) for vk, pi, p in items]
    out += [verify_link_proof(a, b, lp, lay, e.h, e.tau_h) for a, b, lp, lay in links]
    return out


def batch(e, items, links):
    return PlonkKzgSnark.batch_verify(e.ctx, [i[0] for i in items], [i[1] for i in items], [i[2] for i in items], links,
                                      g2=(e.h, e.tau_h))


def proof_items(e, order):
    return [(e.keys[e.proofs[j][0]][1], e.proofs[j][1], e.proofs[j][2]) for j in order]


def test_mixed_batch_is_accepted(env):
    e = env
    # proofs 4, 5 have 120 inputs: 36 copies put 4320 denominators in the batch, more than one 4096-element chunk
    order = [2, 0, 4, 1, 6, 3, 5, 7] + [4, 5] * 18 + [0, 2]
    items = proof_items(e, order)
    assert sum(it[0].num_inputs or 1 for it in items) > 4096
    links = e.links + e.links[:2]
    ok, verdicts = batch(e, items, links)
    assert ok and all(verdicts) and len(verdicts) == len(items) + len(links)
    assert all(single_verdicts(e, items[:8], links))
    ok, verdicts = batch(e, items[:8], [])
    assert ok and all(verdicts)
    ok, verdicts = PlonkKzgSnark.batch_verify(e.ctx, [], [], [], links, g2=(e.h, e.tau_h))
    assert ok and all(verdicts)


def _tamper(e, kind, items, links, pos):
    items, links = list(items), list(links)
    if kind == "link_layout":
        a, b, lp, lay = links[pos]
        links[pos] = (a, b, lp, GroupLayout(lay.alignment, lay.offset + 1, lay.size))
        return items, links
    vk, pi, proof = items[pos]
    p = B200Proof.from_buffer_copy(bytes(proof))
    if kind == "eval_bit":
        p.wires_evals[3][0] ^= 1
    elif kind == "swap_comms":
        w0, w1 = list(p.wires_poly_comms[0]), list(p.wires_poly_comms[1])
        p.wires_poly_comms[0][:], p.wires_poly_comms[1][:] = w1, w0
    elif kind == "pub_input":
        pi = pi.copy()
        pi[0, 0] ^= np.uint64(1)
    elif kind == "wrong_vk":
        wrong = e.keys[3][1] if vk is not e.keys[3][1] else e.keys[1][1]
        assert (wrong.log_n, wrong.num_inputs) == (vk.log_n, vk.num_inputs)
        vk = wrong
    elif kind == "off_curve":
        p.opening_proof[0] ^= 1
    items[pos] = (vk, pi, p)
    return items, links


@pytest.mark.parametrize("kind", ["eval_bit", "swap_comms", "pub_input", "wrong_vk", "off_curve", "link_layout"])
def test_every_tampering_kind_is_located(env, kind):
    e = env
    # first, middle and last proofs are of the 4-input shape, so every kind applies there
    items = proof_items(e, [2, 0, 4, 3, 6, 1, 5, 7, 3])
    n_links = len(e.links)
    positions = [0, n_links // 2, n_links - 1] if kind == "link_layout" else [0, len(items) // 2, len(items) - 1]
    if kind != "link_layout":
        assert all(items[p][0].num_inputs == 4 for p in positions)
    for pos in positions:
        its, lks = _tamper(e, kind, items, e.links, pos)
        want = single_verdicts(e, its, lks)
        assert want.count(False) == 1, (kind, pos)
        ok, verdicts = batch(e, its, lks)
        assert not ok
        assert verdicts == want, (kind, pos)


Q = 21888242871839275222246386852915665306311212217108419009066920287645086208583  # the base field modulus


def _g1_neg(pt):
    q = Q
    y = int.from_bytes(np.asarray(pt[4:8], dtype="<u8").tobytes(), "little")
    out = np.array(pt, dtype=np.uint64).copy()
    out[4:8] = np.frombuffer(((q - y) % q).to_bytes(32, "little"), dtype="<u8")
    return out


def test_randomisers_reject_openings_that_cancel(env):
    """Two link items with the same (C1, C2, Cq, layout), hence the same eta, and openings pi + G and pi - G: each is
    rejected alone and their unweighted sum satisfies the equation (tests/test_batch_verify_cpu.py shows it with the
    oracle's pairing), so only the random weights make the batch reject them."""
    e = env
    a, b, lp, lay = e.links[0]
    q = Q
    mont = lambda v: np.frombuffer(((v << 256) % q).to_bytes(32, "little"), dtype="<u8")
    g = np.concatenate([mont(1), mont(2)]).astype(np.uint64)
    pi = np.array(lp.opening_proof, dtype=np.uint64)
    plus, inf1 = e.ctx.g1_sum_affine(np.stack([pi, g]))
    minus, inf2 = e.ctx.g1_sum_affine(np.stack([pi, _g1_neg(g)]))
    assert not inf1 and not inf2
    lps = []
    for op in (plus, minus):
        x = B200LinkProof.from_buffer_copy(bytes(lp))
        x.opening_proof[:] = [int(v) for v in op]
        lps.append(x)
    pair = [(a, b, x, lay) for x in lps]
    assert single_verdicts(e, [], pair) == [False, False]
    ok, verdicts = PlonkKzgSnark.batch_verify(e.ctx, [], [], [], pair, g2=(e.h, e.tau_h))
    assert not ok and verdicts == [False, False]
    # beside honest items too
    ok, verdicts = batch(e, proof_items(e, [0, 1]), [e.links[1]] + pair + [e.links[2]])
    assert not ok and verdicts == [True, True, True, False, False, True]


def test_identity_selector_commitment(env):
    """A key whose q_ecc column is all zero has the identity as that selector's commitment.  The gates that used q_ecc
    keep their value: q_c absorbs q_ecc * w0 w1 w2 w3 w4 on those rows."""
    e = env
    log_n, ni = 7, 4
    circ = synth.synth_circuit(log_n, num_inputs=ni, seed=21, check=True)
    sel = circ.selectors_int
    rows = [r for r in range(circ.n) if sel[synth.Q_ECC][r]]
    assert rows, "the synthetic circuit uses the ecc gate"
    for r in rows:
        w = [circ.wires_int[j][r] for j in range(5)]
        sel[synth.Q_C][r] = (sel[synth.Q_C][r] + sel[synth.Q_ECC][r] * w[0] * w[1] * w[2] * w[3] * w[4]) % synth.R
        sel[synth.Q_ECC][r] = 0
    for r in range(circ.n):
        pi = circ.pub_inputs_int[r] if r < ni else 0
        assert synth.gate_value([sel[s][r] for s in range(13)], [circ.wires_int[j][r] for j in range(5)], pi) == 0
    selectors = np.stack([synth.to_mont_array(col) for col in sel])
    pk = PlonkKzgSnark.preprocess(e.ctx, e.srs, log_n, ni, selectors, circ.perm, circ.k)
    assert not pk.selector_comms[synth.Q_ECC].any()  # the identity
    vk = VerifyingKey.from_proving_key(pk, e.h, e.tau_h)
    proof, _ = PlonkKzgSnark.prove_with_link_hint(e.ctx, pk, circ.wires, circ.pub_inputs, synth.splitmix_blinders(5))
    items = [(vk, circ.pub_inputs, proof)] + proof_items(e, [2, 3]) + [(vk, circ.pub_inputs, proof)]
    assert all(single_verdicts(e, items, []))
    ok, verdicts = batch(e, items, [])
    assert ok and all(verdicts)
    bad = B200Proof.from_buffer_copy(bytes(proof))
    bad.wires_evals[0][0] ^= 1
    items[3] = (vk, circ.pub_inputs, bad)
    ok, verdicts = batch(e, items, [])
    assert not ok and verdicts == single_verdicts(e, items, []) == [True, True, True, False]
    pk.free()


def test_sizes_and_permutation(env):
    e = env
    ok, verdicts = PlonkKzgSnark.batch_verify(e.ctx, [], [], [], [], g2=(e.h, e.tau_h))
    assert ok and verdicts == []
    for order in ([2], [2, 5]):
        ok, verdicts = batch(e, proof_items(e, order), [])
        assert ok and verdicts == [True] * len(order)
    base = proof_items(e, [0, 1, 2, 3, 6, 7])
    items = [base[i % len(base)] for i in range(4095)]
    vk, pi, proof = items[0]
    bad = B200Proof.from_buffer_copy(bytes(proof))
    bad.wires_evals[1][2] ^= 1
    assert not PlonkKzgSnark.verify(vk, pi, bad)
    items.append((vk, pi, bad))
    ok, verdicts = batch(e, items, [])
    assert not ok and verdicts == [True] * 4095 + [False]
    perm = list(range(4096))
    random.Random(4096).shuffle(perm)
    ok, pv = batch(e, [items[i] for i in perm], [])
    assert not ok and pv == [verdicts[i] for i in perm]
    # a wrong public-input count is a False verdict, as for the single verifier
    vk2, pi2, p2 = base[2]
    ok, verdicts = batch(e, [base[0], (vk2, pi2[:-1], p2)], [])
    assert not ok and verdicts == [True, False]


def test_mismatched_g2_pairs_are_refused(env):
    e = env
    vk = e.keys[1][1]
    other = VerifyingKey(vk.log_n, vk.num_inputs, vk.k, vk.selector_comms, vk.sigma_comms, e.tau_h, e.h)
    with pytest.raises(ValueError):
        PlonkKzgSnark.batch_verify(e.ctx, [vk, other], [e.proofs[2][1]] * 2, [e.proofs[2][2]] * 2)


def test_real_statements(ctx, srs_2_16, srs_2_16_g2):
    from host_circuits import intent_and_balance_validity as val
    from host_circuits import statements as st
    from host_circuits import valid_balance_create as vbc
    from renegade_b200 import circuit_types as ct
    params = rb.parse_ptau_file(ctx, srs_2_16, count=(1 << 16) + 3)
    h, tau_h = srs_2_16_g2
    ct.set_system_srs(ctx, params.powers_of_g, h, tau_h)
    try:
        batch_items = []
        for seed in (7, 8):
            w, s = vbc.create_witness_statement(seed)
            batch_items.append((st.ValidBalanceCreate, s, ct.singleprover_prove(st.ValidBalanceCreate, w, s)))
        w, s = val.create_witness_statement(seed=70)
        batch_items.append((st.IntentAndBalanceValidityCircuit, s,
                            ct.singleprover_prove(st.IntentAndBalanceValidityCircuit, w, s)))
        ct.batch_verify_singleprover_proofs(batch_items)
        for c, s, p in batch_items:
            ct.verify_singleprover_proof(c, s, p)
        wrong = list(batch_items)
        wrong[1] = (wrong[1][0], batch_items[0][1], wrong[1][2])  # proof 1 under statement 0
        with pytest.raises(ct.VerifierError) as err:
            ct.batch_verify_singleprover_proofs(wrong)
        assert "[1]" in str(err.value)
    finally:
        ct.clear_key_cache()
