"""CPU evidence for the batch verifier's random weights (tests/test_gpu_batch_verify.py::
test_randomisers_reject_openings_that_cancel): two link proofs that share (C1, C2, Cq, layout) and open with pi + G and
pi - G each fail the link equation, but their UNWEIGHTED sum satisfies it.  Restated here in Python on the oracle's
link proof and its pure-Python pairing: with weights (1, 1) the batched equation accepts the pair, with two different
weights it rejects it.  Also: the new entry point and its structs are part of the header, the binding list and the
Rust FFI that tests/test_abi_cpu.py checks against each other."""
import os
import re

import numpy as np

from renegade_b200 import _lib, synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _link_fixture(oracle, py, srs_head):
    layout = (5, 6, 5)  # alignment, offset, size
    vals = [(i * 1234567 + 89) % py.R for i in range(layout[2])]
    hints = []
    for log_n, seed in ((6, 3), (7, 4)):
        n = 1 << log_n
        circ = synth.synth_circuit(log_n, num_inputs=2, seed=seed, check=True, link=(layout[0], layout[1], vals))
        srs = np.frombuffer(srs_head[80:80 + 64 * (n + 3)], dtype=np.uint64).reshape(n + 3, 8).copy()
        pk = oracle.plonk_preprocess(log_n, circ.selectors, circ.perm, circ.k, srs)
        rc, proof, _, link = oracle.plonk_prove(log_n, circ.num_inputs, circ.k, pk, circ.wires, circ.pub_inputs,
                                                synth.splitmix_blinders(seed), srs, True)
        assert rc == 0
        hints.append((link, np.array(proof.wires_poly_comms[0], dtype=np.uint64)))
    srs_all = np.frombuffer(srs_head[80:], dtype=np.uint64).reshape(-1, 8)
    rc, lp, eta = oracle.plonk_link(hints[0][0], hints[1][0], hints[0][1], hints[1][1], *layout, srs_all)
    assert rc == 0
    return layout, hints[0][1], hints[1][1], lp, eta


def test_cancelling_openings_pass_unweighted_and_fail_weighted(oracle, pyoracle, srs_head, g2_raw):
    import bn254_pairing_py as pr
    py = pyoracle
    layout, c1_raw, c2_raw, lp, eta_mont = _link_fixture(oracle, py, srs_head)
    dec = lambda a: py.decode_g1_mont(np.ascontiguousarray(a, dtype=np.uint64).tobytes(), 0)
    c1, c2 = dec(c1_raw), dec(c2_raw)
    cq, pi = dec(lp.quotient_commitment), dec(lp.opening_proof)
    eta = py.from_mont(int.from_bytes(np.ascontiguousarray(eta_mont, dtype=np.uint64).tobytes(), "little"), py.R)
    alignment, offset, size = layout
    g = py.domain_generator(alignment)
    zd = 1
    for i in range(size):
        zd = zd * (eta - pow(g, offset + i, py.R)) % py.R
    G = (1, 2)
    openings = [py.g1_add(pi, G), py.g1_add(pi, py.g1_neg(G))]
    raw = g2_raw[0].tobytes() + g2_raw[1].tobytes()
    h, tau_h = pr.decode_g2_mont(raw, 0), pr.decode_g2_mont(raw, 1)
    x = py.g1_add(py.g1_add(c1, py.g1_neg(c2)), py.g1_neg(py.g1_mul(cq, zd)))  # C1 - C2 - Z_D(eta) Cq

    def batched(weights):
        """e(sum rho_i pi_i, [tau]_2) == e(sum rho_i (X + eta pi_i), [1]_2)"""
        a = b = None
        for rho, op in zip(weights, openings):
            a = py.g1_add(a, py.g1_mul(op, rho))
            b = py.g1_add(b, py.g1_mul(py.g1_add(x, py.g1_mul(op, eta)), rho))
        return pr.pairing_product_is_one([(a, tau_h), (py.g1_neg(b) if b is not None else None, h)])

    assert batched([1, 1])      # the openings' errors cancel: an unweighted sum accepts the pair
    assert not batched([1, 2])  # two different weights expose them


def test_batch_entry_point_is_in_header_binding_and_ffi():
    header = open(os.path.join(ROOT, "include", "b200prover.h")).read()
    ffi = open(os.path.join(ROOT, "shim", "gpu-prover", "src", "ffi.rs")).read()
    assert re.search(r"\bint b200_plonk_batch_verify\(", header)
    assert "b200_plonk_batch_verify" in _lib.EXPORTS
    assert "pub fn b200_plonk_batch_verify(" in ffi
    for struct in ("b200_verifying_key", "b200_batch_proof", "b200_batch_link"):
        assert re.search(r"\}\s*" + struct + ";", header), struct
        assert "pub struct " + struct in ffi, struct
