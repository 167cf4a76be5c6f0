"""The host verifiers (`b200_plonk_verify`, `b200_plonk_verify_link`, `b200_pairing_check`) field by field: every
mutation of `verify_mutations.py` — each proof point, evaluation and public input, each verifying-key field, each part
of a link proof and its layout, into an encoding outside the field or into a wrong canonical value — is rejected.

The ABI takes Montgomery limbs a 2^256 mod p, so an element's only valid encoding lies in [0, p).  The transcript
hashes reduced values and the multiplier reduces its operands, so v + p would otherwise verify as v: a second
encoding of an honest proof the reference (arkworks refuses a field element >= p when it deserializes) never accepts.

Proofs come from the oracle prover on the reference's SRS head (tests/golden/srs_head.bin) and its G2 pair."""
import numpy as np
import pytest

import verify_mutations as vm
from renegade_b200 import _lib, synth
from renegade_b200.backend import (B200LinkProof, B200Proof, GroupLayout, PlonkKzgSnark, VerifyingKey, pairing_check,
                                   verify_link_proof)

LOG_N, NUM_INPUTS = 7, 4
LAYOUT = (5, 6, 5)  # alignment, offset, size
B200_ERR_NOT_ON_CURVE = -5


class Env:
    pass


@pytest.fixture(scope="module")
def env(oracle, pyoracle, srs_head, g2_raw):
    e = Env()
    e.h, e.tau_h = g2_raw
    vals = [(i * 7654321 + 5) % pyoracle.R for i in range(LAYOUT[2])]
    hints = []
    for log_n, ni, seed in ((LOG_N, NUM_INPUTS, 31), (6, 2, 3)):
        n = 1 << log_n
        circ = synth.synth_circuit(log_n, num_inputs=ni, seed=seed, check=True, link=(LAYOUT[0], LAYOUT[1], vals))
        srs = np.frombuffer(srs_head[80:80 + 64 * (n + 3)], dtype=np.uint64).reshape(n + 3, 8).copy()
        pk = oracle.plonk_preprocess(log_n, circ.selectors, circ.perm, circ.k, srs)
        rc, proof, _, link = oracle.plonk_prove(log_n, ni, circ.k, pk, circ.wires, circ.pub_inputs,
                                                synth.splitmix_blinders(seed), srs, True)
        assert rc == 0
        hints.append((link, np.array(proof.wires_poly_comms[0], dtype=np.uint64)))
        if log_n == LOG_N:
            e.plonk = vm.PlonkItem(circ.k, pk["selector_comms"], pk["sigma_comms"], circ.pub_inputs, proof.to_array())
    srs_all = np.frombuffer(srs_head[80:], dtype=np.uint64).reshape(-1, 8)
    rc, lp, _ = oracle.plonk_link(hints[1][0], hints[0][0], hints[1][1], hints[0][1], *LAYOUT, srs_all)
    assert rc == 0
    e.link = vm.LinkItem(hints[1][1], hints[0][1], lp.to_array(), LAYOUT)
    e.plonk_muts = vm.plonk_mutations(e.plonk)
    e.link_muts = vm.link_mutations(e.link)
    return e


def verify_plonk(e, it: vm.PlonkItem) -> bool:
    vk = VerifyingKey(LOG_N, NUM_INPUTS, it.k, it.sel, it.sig, e.h, e.tau_h)
    return PlonkKzgSnark.verify(vk, it.pi, B200Proof.from_buffer_copy(it.proof.tobytes()))


def verify_link(e, it: vm.LinkItem) -> bool:
    return verify_link_proof(it.c1, it.c2, B200LinkProof.from_buffer_copy(it.lp.tobytes()), GroupLayout(*it.layout),
                             e.h, e.tau_h)


def test_mutation_matrix_covers_every_field(env):
    e = env
    labels = [m.label for m in e.plonk_muts + e.link_muts]
    assert len(set(labels)) == len(labels)
    # a point: x and y each outside the field three ways, and up to four wrong points; a scalar: six values
    fields = {}
    for m in e.plonk_muts + e.link_muts:
        fields.setdefault(m.label.split(".x:")[0].split(".y:")[0].split(":")[0], set()).add(m.cls)
    points = ([f"proof.{n}" for n, _ in vm.PROOF_POINTS] + [f"vk.selector_comms[{i}]" for i in range(13)] +
              [f"vk.sigma_comms[{i}]" for i in range(5)] + ["link.comm1", "link.comm2", "link.quotient_commitment",
                                                            "link.opening_proof"])
    scalars = ([f"proof.{n}" for n, _ in vm.PROOF_EVALS] + [f"pi[{i}]" for i in range(NUM_INPUTS)] +
               [f"vk.k[{i}]" for i in range(5)])
    for f in points:
        assert set(vm.NON_CANONICAL) | {"neg", "double", "generator"} <= fields[f], f
    for f in scalars:
        assert set(vm.NON_CANONICAL) | {"minus_one", "plus_one"} <= fields[f], f
    # alignment, offset and size each move both ways at this layout
    assert sum(m.cls == vm.LAYOUT for m in e.link_muts) == 6
    assert set(fields) - {m.label for m in e.link_muts if m.cls == vm.LAYOUT} == set(points) | set(scalars)


def test_honest_items_are_accepted(env):
    assert verify_plonk(env, env.plonk)
    assert verify_link(env, env.link)


def test_every_proof_mutation_is_rejected(env):
    accepted = [m.label for m in env.plonk_muts if verify_plonk(env, m.item)]
    assert accepted == []


def test_every_link_mutation_is_rejected(env):
    accepted = [m.label for m in env.link_muts if verify_link(env, m.item)]
    assert accepted == []


def test_canonical_mutations_agree_with_the_oracle(env, oracle):
    """One mutation per canonical class, each on another kind of field, through the oracle's verifier and the
    independent Python pairing: it rejects them too (and accepts the honest proof)."""
    import bn254_pairing_py as pr
    e = env
    raw = e.h.tobytes() + e.tau_h.tobytes()
    g2 = (pr.decode_g2_mont(raw, 0), pr.decode_g2_mont(raw, 1))
    picks = ["proof.wires_poly_comms[2]:identity", "vk.selector_comms[4]:neg", "proof.opening_proof:double",
             "vk.sigma_comms[1]:generator", "proof.wire_sigma_evals[2]:zero", "pi[1]:minus_one", "vk.k[3]:plus_one"]
    by_label = {m.label: m for m in e.plonk_muts}
    assert {by_label[p].cls for p in picks} == set(vm.POINT_VALUES + vm.SCALAR_VALUES)

    def oracle_verify(it):
        proof = oracle.PlonkProof.from_buffer_copy(it.proof.tobytes())
        return oracle.plonk_verify_pairing(LOG_N, NUM_INPUTS, it.k, {"selector_comms": it.sel, "sigma_comms": it.sig},
                                           it.pi, proof, *g2)
    assert oracle_verify(e.plonk)
    for p in picks:
        it = by_label[p].item
        assert not oracle_verify(it), p
        assert not verify_plonk(e, it), p


def test_pairing_check_refuses_non_canonical_coordinates(env, pyoracle):
    """`b200_pairing_check` refuses a coordinate >= q in G1 or G2 as it refuses an off-curve point; the single verifiers
    refuse such a G2 record the same way (an error, not a rejection)."""
    e = env
    py = pyoracle
    g = np.frombuffer(py.encode_g1_mont(py.G1_GEN), dtype=np.uint64).copy()
    ng = np.frombuffer(py.encode_g1_mont(py.g1_neg(py.G1_GEN)), dtype=np.uint64).copy()
    assert pairing_check([g, ng], [e.h, e.h])

    def bumped(words, j, enc):
        w = np.array(words, dtype=np.uint64)
        w[4 * j:4 * j + 4] = vm.to_words(enc)
        return w

    def refused(g1s, g2s):
        with pytest.raises(_lib.B200Error) as err:
            pairing_check(g1s, g2s)
        return err.value.code == B200_ERR_NOT_ON_CURVE

    for j in range(2):  # x, y of G and of the identity
        for base in (g, np.zeros(8, dtype=np.uint64)):
            for enc in vm.out_of_field(vm.to_int(base[4 * j:4 * j + 4]), vm.Q).values():
                assert refused([bumped(base, j, enc), ng], [e.h, e.h]), (j, enc)
    for j in range(4):  # x0, x1, y0, y1 of h
        for enc in vm.out_of_field(vm.to_int(e.h[4 * j:4 * j + 4]), vm.Q).values():
            bad_h = bumped(e.h, j, enc)
            assert refused([g, ng], [bad_h, e.h]), (j, enc)
            vk = VerifyingKey(LOG_N, NUM_INPUTS, e.plonk.k, e.plonk.sel, e.plonk.sig, bad_h, e.tau_h)
            with pytest.raises(_lib.B200Error) as err:
                PlonkKzgSnark.verify(vk, e.plonk.pi, B200Proof.from_buffer_copy(e.plonk.proof.tobytes()))
            assert err.value.code == B200_ERR_NOT_ON_CURVE
            with pytest.raises(_lib.B200Error) as err:
                verify_link_proof(e.link.c1, e.link.c2, B200LinkProof.from_buffer_copy(e.link.lp.tobytes()),
                                  GroupLayout(*e.link.layout), e.h, bad_h)
            assert err.value.code == B200_ERR_NOT_ON_CURVE
