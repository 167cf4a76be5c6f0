"""Proving from the witness vector, the parts that need no GPU: the new entry points in the header, the binding and the
Rust shim agree; the rule by which `b200_plonk_preprocess_wiring` derives the copy permutation, restated in numpy, has
exactly the variables' position sets as its cycles; and the circuit-as-(wiring, witness) fixtures expand to the value
tables the oracle prover accepts.  `wiring_permutation` here is the reference tests/test_gpu_prove_witness.py uses."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from renegade_b200 import synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW = ["b200_plonk_preprocess_wiring", "b200_pk_num_vars", "b200_plonk_prove_witness", "b200_plonk_prove_witness_batch",
       "b200_pool_submit_prove_witness"]


def wiring_permutation(wire_vars) -> np.ndarray:
    """The positions p = i*n + j of one variable, in ascending p, form one cycle: each maps to the next, the last to
    the first."""
    v = np.asarray(wire_vars, dtype=np.uint32).reshape(-1)
    order = np.argsort(v, kind="stable")              # grouped by variable, ascending position inside a group
    sv = v[order]
    nxt = np.roll(order, -1)
    last = np.r_[sv[1:] != sv[:-1], True]             # last position of its group
    first = order[np.r_[True, sv[1:] != sv[:-1]]]     # first position of every group, in group order
    nxt[last] = first
    perm = np.empty(v.size, dtype=np.uint64)
    perm[order] = nxt
    return perm


def expand(circ) -> np.ndarray:
    """The 5 x n value table of a circuit given as wiring + witness vector."""
    return circ.witness[circ.wire_vars]


def cycles(perm) -> set:
    seen, out = np.zeros(len(perm), dtype=bool), set()
    for p in range(len(perm)):
        if not seen[p]:
            cyc, q = [], p
            while not seen[q]:
                seen[q] = True
                cyc.append(q)
                q = int(perm[q])
            out.add(frozenset(cyc))
    return out


def test_new_entry_points_in_header_binding_and_shim():
    from renegade_b200 import _lib
    _, structs, funcs, _ = _lib.parse_header()
    sig = {name: (ret, args) for name, ret, args in funcs}
    assert all(n in _lib.EXPORTS for n in NEW)
    assert sig["b200_pk_num_vars"] == ("size_t", [("pk", "const b200_pk *")])
    assert [a for a, _ in sig["b200_plonk_preprocess_wiring"][1]] == [
        "ctx", "srs", "log_n", "num_inputs", "selectors_evals", "wire_vars", "num_vars", "k", "out"]
    assert dict(sig["b200_plonk_preprocess_wiring"][1])["wire_vars"] == "const unsigned *"
    assert [a for a, _ in sig["b200_plonk_prove_witness"][1]] == [
        "ctx", "pk", "witness", "blinders", "proof", "link_poly", "challenges", "pub_inputs_out"]
    assert [a for a, _ in sig["b200_pool_submit_prove_witness"][1]] == [
        "pool", "pk", "witness", "blinders", "proof", "link_poly", "pub_inputs_out", "ticket"]
    assert [f for f, _, _ in structs["b200_witness_item"]] == ["witness", "blinders", "proof", "link_poly", "challenges",
                                                             "pub_inputs_out"]
    item = _lib.STRUCTS["b200_witness_item"]
    assert C.sizeof(item) == 6 * C.sizeof(C.c_void_p)
    lib = _lib.load()  # every declared symbol is exported, with the header's signature
    assert lib.b200_plonk_prove_witness.argtypes == [C.c_void_p] * 8
    assert lib.b200_pk_num_vars.restype is C.c_size_t
    assert lib.b200_pk_num_vars(None) == 0
    ffi = open(os.path.join(ROOT, "shim", "gpu-prover", "src", "ffi.rs")).read()
    for n in NEW:
        assert re.search(rf"pub fn {n}\(", ffi), n
    assert "pub struct b200_witness_item" in ffi
    shim = open(os.path.join(ROOT, "shim", "gpu-prover", "src", "lib.rs")).read()
    assert "ffi::b200_plonk_preprocess_wiring(" in shim and "ffi::b200_pool_submit_prove_witness(" in shim


def test_null_arguments_are_refused_without_a_device():
    from renegade_b200 import _lib
    lib = _lib.load()
    h = C.c_void_p()
    assert lib.b200_plonk_preprocess_wiring(None, None, 4, 0, None, None, 1, None, C.byref(h)) == _lib.B200_ERR_INVALID
    assert lib.b200_plonk_prove_witness(None, None, None, None, None, None, None, None) == _lib.B200_ERR_INVALID
    assert lib.b200_plonk_prove_witness_batch(None, None, None, 0, None) == _lib.B200_ERR_INVALID
    t = C.c_uint64()
    assert lib.b200_pool_submit_prove_witness(None, None, None, None, None, None, None, C.byref(t)) == _lib.B200_ERR_INVALID


@pytest.mark.parametrize("log_n,link", [(4, False), (7, True), (10, False)])
def test_permutation_rule_has_the_variables_as_cycles(log_n, link):
    lk = (log_n - 1, 2, [5, 6, 7]) if link else None
    circ = synth.synth_circuit(log_n, num_inputs=2, seed=90 + log_n, link=lk)
    assert circ.wire_vars.shape == (5, circ.n) and circ.wire_vars.dtype == np.uint32
    assert circ.witness.shape == (circ.num_vars, 4) and int(circ.wire_vars.max()) < circ.num_vars
    perm = wiring_permutation(circ.wire_vars)
    assert sorted(perm.tolist()) == list(range(5 * circ.n))  # a permutation
    flat = circ.wire_vars.reshape(-1)
    want = {frozenset(np.flatnonzero(flat == v).tolist()) for v in np.unique(flat)}
    assert cycles(perm) == want
    # SynthCircuit.perm walks each variable's positions in row-major order: another permutation, the same cycle sets
    assert cycles(circ.perm) == want
    assert (flat[perm.astype(np.int64)] == flat).all()
    # every position maps to the next higher one of its variable, the highest to the lowest
    up = perm.astype(np.int64) > np.arange(5 * circ.n)
    assert (~up).sum() == len(want)
    # the expanded table is the circuit's, and the public inputs sit on the output wire of the first rows
    assert (expand(circ) == circ.wires).all()
    assert (circ.witness[circ.wire_vars[4, :circ.num_inputs]] == circ.pub_inputs).all()


def test_permutation_rule_edges():
    assert wiring_permutation(np.zeros(20, dtype=np.uint32)).tolist() == list(range(1, 20)) + [0]
    assert wiring_permutation(np.arange(20, dtype=np.uint32)[::-1]).tolist() == list(range(20))  # every variable once
    assert wiring_permutation(np.array([7, 3, 7, 3, 9], dtype=np.uint32)).tolist() == [2, 3, 0, 1, 4]


def test_oracle_proves_the_expanded_table_under_the_derived_permutation(oracle, pyoracle):
    py = pyoracle
    log_n = 5
    circ = synth.synth_circuit(log_n, num_inputs=2, seed=17, check=True)
    tau = oracle.int_to_limbs(py.to_mont(0xB200B200 % py.R, py.R))
    srs = oracle.srs_from_tau(tau, circ.n + 3)
    perm = wiring_permutation(circ.wire_vars)
    opk = oracle.plonk_preprocess(log_n, circ.selectors, perm, circ.k, srs)
    wires = np.ascontiguousarray(expand(circ))
    pub = np.ascontiguousarray(circ.witness[circ.wire_vars[4, :circ.num_inputs]])
    bl = synth.splitmix_blinders(3)
    rc, proof, _, _ = oracle.plonk_prove(log_n, circ.num_inputs, circ.k, opk, wires, pub, bl, srs)
    assert rc == 0
    assert oracle.plonk_verify_known_tau(log_n, circ.num_inputs, circ.k, opk, pub, proof, tau)
    bad = wires.copy()
    bad[4, circ.num_inputs + 1] = bad[4, circ.num_inputs + 2]
    assert oracle.plonk_prove(log_n, circ.num_inputs, circ.k, opk, bad, pub, bl, srs)[0] != 0


def test_host_constraint_system_gives_wiring_and_witness():
    from host_circuits import circuit as hc
    import random
    rnd = random.Random(5)
    leaf = [rnd.randrange(hc.R) for _ in range(4)]
    opening = hc.MerkleOpening([rnd.randrange(hc.R) for _ in range(2)], [True, False])
    full = hc.merkle_membership_circuit(leaf, opening)[0].finalize_for_arithmetization()
    assert (expand(full) == full.wires).all() and full.num_vars == len(full.witness)
    assert cycles(wiring_permutation(full.wire_vars)) == cycles(full.perm)
    lean = hc.merkle_membership_circuit(leaf, opening)[0].finalize_for_arithmetization(witness_only=True)
    assert lean.wires is None and lean.perm is None and lean.selectors is None
    assert (lean.witness == full.witness).all() and (lean.pub_inputs == full.pub_inputs).all()
    assert lean.structure_digest == full.structure_digest and lean.log_n == full.log_n
