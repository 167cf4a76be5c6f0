"""GPU parity: the TurboPlonk prover rounds on the device vs the CPU restatement — same SRS, same
witness, same 17 blinding scalars => byte-identical proof (every commitment, evaluation and
Fiat–Shamir challenge), accepted by the (restated) verifier; an unsatisfying witness is rejected
like the reference's WrongQuotientPolyDegree."""
import numpy as np
import pytest

import renegade_b200 as rb
from renegade_b200 import synth
from renegade_b200.backend import PlonkKzgSnark

pytestmark = pytest.mark.gpu

TAU = 0x2f1a6c0b5d3e49788a9bc0d1e2f30415263748596a7b8c9dae0f1f2e3d4c5b6a


def setup(ctx, oracle, pyoracle, log_n, seed, num_inputs=7):
    py = pyoracle
    n = 1 << log_n
    circ = synth.synth_circuit(log_n, num_inputs=num_inputs, seed=seed, check=(log_n <= 10))
    tau = oracle.int_to_limbs(py.to_mont(TAU % py.R, py.R))
    srs = oracle.srs_from_tau(tau, n + 3)
    return circ, tau, srs


# every domain from 2^5 to 2^15: the chunked scans (CH = 16) change their level structure across these sizes, e.g. 16,
# 256 and 4096 chunks fill a top level exactly
@pytest.mark.parametrize("log_n", [5, 7, 8, 9, 10, 11, 12, 13, 14, 15])
def test_prove_matches_oracle_bit_exact(ctx, oracle, pyoracle, log_n):
    circ, tau, srs = setup(ctx, oracle, pyoracle, log_n, seed=100 + log_n)
    bases = ctx.load_bases(srs, check_on_curve=True)
    pk = PlonkKzgSnark.preprocess(ctx, bases, log_n, circ.num_inputs, circ.selectors, circ.perm, circ.k)
    opk = oracle.plonk_preprocess(log_n, circ.selectors, circ.perm, circ.k, srs)
    assert (pk.selector_comms == opk["selector_comms"]).all()
    assert (pk.sigma_comms == opk["sigma_comms"]).all()
    blinders = synth.splitmix_blinders(0xB11D + log_n)
    proof, hint, ch = PlonkKzgSnark.prove_with_link_hint(ctx, pk, circ.wires, circ.pub_inputs, blinders, want_challenges=True)
    rc, oproof, och, olink = oracle.plonk_prove(log_n, circ.num_inputs, circ.k, opk, circ.wires, circ.pub_inputs, blinders, srs, True)
    assert rc == 0
    ours, theirs = proof.to_array(), oproof.to_array()
    names = ["wire_comm"] * 40 + ["z_comm"] * 8 + ["quot_comm"] * 40 + ["opening"] * 8 + ["shifted"] * 8 + \
            ["wire_eval"] * 20 + ["sigma_eval"] * 16 + ["z_next"] * 4
    diff = [names[i] for i in range(len(names)) if ours[i] != theirs[i]]
    assert not diff, sorted(set(diff))
    assert (ch.reshape(-1) == np.frombuffer(bytes(och), dtype=np.uint64)).all()
    assert (hint.linking_wire_poly == olink).all()
    assert (hint.linking_wire_comm == ours[:8]).all()
    if log_n == 5:  # the committed proof fixture was cut with exactly these parameters (tests/golden/make_proof_golden.py)
        import hashlib
        import json
        import os
        with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "proof_kat.json")) as f:
            want = json.load(f)
        assert (want["params"]["circuit_seed"], want["params"]["blinder_seed"], int(want["params"]["tau"], 16)) == (105, 0xB11D + 5, TAU)
        assert bytes(proof).hex() == want["proof_hex"]
        assert hashlib.sha256(np.ascontiguousarray(hint.linking_wire_poly).tobytes()).hexdigest() == want["link_poly_sha256"]
        assert hashlib.sha256(pk.selector_comms.tobytes() + pk.sigma_comms.tobytes()).hexdigest() == want["vk_sha256"]
    # the restated verifier accepts the device proof; tampering is rejected
    op = oracle.PlonkProof.from_buffer_copy(bytes(proof))
    assert oracle.plonk_verify_known_tau(log_n, circ.num_inputs, circ.k, opk, circ.pub_inputs, op, tau)
    op.wires_evals[2][0] ^= 1
    assert not oracle.plonk_verify_known_tau(log_n, circ.num_inputs, circ.k, opk, circ.pub_inputs, op, tau)


def test_unsatisfied_witness_rejected(ctx, oracle, pyoracle):
    from renegade_b200._lib import B200Error
    log_n = 9
    circ, tau, srs = setup(ctx, oracle, pyoracle, log_n, seed=5)
    bases = ctx.load_bases(srs)
    pk = PlonkKzgSnark.preprocess(ctx, bases, log_n, circ.num_inputs, circ.selectors, circ.perm, circ.k)
    bad = circ.wires.copy()
    bad[4, circ.num_inputs + 3] = bad[4, circ.num_inputs + 4]
    with pytest.raises(B200Error) as ei:
        PlonkKzgSnark.prove_with_link_hint(ctx, pk, bad, circ.pub_inputs, synth.splitmix_blinders(1))
    assert ei.value.code == -7 and "WrongQuotientPolyDegree" in str(ei.value)
    # the same key still proves a good witness afterwards
    proof, _ = PlonkKzgSnark.prove_with_link_hint(ctx, pk, circ.wires, circ.pub_inputs, synth.splitmix_blinders(1))
    opk = {"selector_comms": pk.selector_comms, "sigma_comms": pk.sigma_comms}
    assert oracle.plonk_verify_known_tau(log_n, circ.num_inputs, circ.k, opk, circ.pub_inputs,
                                         oracle.PlonkProof.from_buffer_copy(bytes(proof)), tau)


def test_prove_2_16_verifies(ctx, oracle, pyoracle):
    """The '~2^16 constraints' configuration (BASELINE.json configs[3]) at full size: device proof
    accepted by the restated verifier, and equal to the oracle's proof."""
    log_n = 16
    circ, tau, srs = setup(ctx, oracle, pyoracle, log_n, seed=0xB200, num_inputs=17)
    bases = ctx.load_bases(srs)
    pk = PlonkKzgSnark.preprocess(ctx, bases, log_n, circ.num_inputs, circ.selectors, circ.perm, circ.k)
    blinders = synth.splitmix_blinders(0x5EED)
    proof, hint = PlonkKzgSnark.prove_with_link_hint(ctx, pk, circ.wires, circ.pub_inputs, blinders)
    opk = oracle.plonk_preprocess(log_n, circ.selectors, circ.perm, circ.k, srs)
    assert (pk.selector_comms == opk["selector_comms"]).all() and (pk.sigma_comms == opk["sigma_comms"]).all()
    op = oracle.PlonkProof.from_buffer_copy(bytes(proof))
    assert oracle.plonk_verify_known_tau(log_n, circ.num_inputs, circ.k, opk, circ.pub_inputs, op, tau)
    rc, oproof, _, _ = oracle.plonk_prove(log_n, circ.num_inputs, circ.k, opk, circ.wires, circ.pub_inputs, blinders, srs)
    assert rc == 0 and (proof.to_array() == oproof.to_array()).all()


def test_prove_2_17_max_domain(ctx, oracle, pyoracle):
    """The largest domain the reference supports: MAX_SRS_DEGREE = 2^17 + 2 (srs.rs:44-47), i.e. an
    SRS of exactly 2^17 + 3 powers and blinded polynomials of n + 3 coefficients."""
    log_n = 17
    circ, tau, srs = setup(ctx, oracle, pyoracle, log_n, seed=0x17, num_inputs=13)
    assert srs.shape[0] == (1 << 17) + 3
    bases = ctx.load_bases(srs)
    pk = PlonkKzgSnark.preprocess(ctx, bases, log_n, circ.num_inputs, circ.selectors, circ.perm, circ.k)
    blinders = synth.splitmix_blinders(0x1717)
    proof, hint = PlonkKzgSnark.prove_with_link_hint(ctx, pk, circ.wires, circ.pub_inputs, blinders)
    opk = {"selector_comms": pk.selector_comms, "sigma_comms": pk.sigma_comms}
    op = oracle.PlonkProof.from_buffer_copy(bytes(proof))
    assert oracle.plonk_verify_known_tau(log_n, circ.num_inputs, circ.k, opk, circ.pub_inputs, op, tau)
    # one more power than the SRS holds must be refused up front (MAX_SRS_DEGREE rule), not crash
    from renegade_b200._lib import B200Error
    short = ctx.load_bases(srs[: (1 << 17) + 2])
    with pytest.raises(B200Error):
        PlonkKzgSnark.preprocess(ctx, short, log_n, circ.num_inputs, circ.selectors, circ.perm, circ.k)


def test_zero_public_inputs_and_tiny_domain(ctx, oracle, pyoracle):
    """Edge cases: a circuit without public inputs, the smallest domain the prover accepts (n = 4), and the
    domains either side of the switch from 8 to 6 quotient cosets (n = 8 -> 8 cosets, n = 16 -> 6: 6n exceeds the
    quotient's 5n + 8 coefficients by only 8 there)."""
    for log_n, num_inputs in ((6, 0), (2, 1), (3, 2), (4, 3)):
        circ, tau, srs = setup(ctx, oracle, pyoracle, log_n, seed=40 + log_n, num_inputs=num_inputs)
        bases = ctx.load_bases(srs)
        pk = PlonkKzgSnark.preprocess(ctx, bases, log_n, circ.num_inputs, circ.selectors, circ.perm, circ.k)
        bl = synth.splitmix_blinders(3)
        proof, _ = PlonkKzgSnark.prove_with_link_hint(ctx, pk, circ.wires, circ.pub_inputs, bl)
        opk = oracle.plonk_preprocess(log_n, circ.selectors, circ.perm, circ.k, srs)
        rc, oproof, _, _ = oracle.plonk_prove(log_n, circ.num_inputs, circ.k, opk, circ.wires, circ.pub_inputs, bl, srs)
        assert rc == 0 and (proof.to_array() == oproof.to_array()).all(), (log_n, num_inputs)
        assert oracle.plonk_verify_known_tau(log_n, circ.num_inputs, circ.k, opk, circ.pub_inputs, oproof, tau)
