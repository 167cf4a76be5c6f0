"""The shapes of tests/witness_shapes.py on the host alone: each builder has the sort width, top-bit pairs, cycle
structure, gates and public inputs it claims, and on the small shapes the oracle proves the expanded table under the
permutation the wiring implies (rc 0) and verifies the proof.  tests/test_gpu_witness_shapes.py asserts the same
preconditions before it compares the device's keys and proofs."""
import numpy as np
import pytest

import witness_shapes as ws
from renegade_b200 import synth
from test_prove_witness_cpu import cycles, expand, wiring_permutation

RINV = pow(1 << 256, -1, synth.R)


def position_sets(wire_vars) -> set:
    """Each variable's positions in the flattened 5 x n wiring."""
    v = np.asarray(wire_vars, dtype=np.uint32).reshape(-1)
    order = np.argsort(v, kind="stable")
    cuts = np.flatnonzero(v[order][1:] != v[order][:-1]) + 1
    return {frozenset(g.tolist()) for g in np.split(order, cuts)}


def to_int(limbs) -> int:
    return int.from_bytes(np.ascontiguousarray(limbs, dtype=np.uint64).tobytes(), "little") * RINV % synth.R


def assert_gates_and_public_inputs(circ):
    """Every row's TurboPlonk gate holds on the expanded table (rows with zero selectors past the public inputs hold
    trivially), and the public inputs are the output-wire values of the first num_inputs rows."""
    ni = circ.num_inputs
    wires = expand(circ)
    assert (circ.pub_inputs == circ.witness[circ.wire_vars[4, :ni]]).all()
    live = np.flatnonzero(circ.selectors.any(axis=(0, 2)))
    for j in sorted(set(live.tolist()) | set(range(ni))):
        q = [to_int(circ.selectors[s, j]) for s in range(synth.N_SELECTORS)]
        w = [to_int(wires[i, j]) for i in range(synth.N_WIRES)]
        pi = to_int(circ.pub_inputs[j]) if j < ni else 0
        assert synth.gate_value(q, w, pi) == 0, j


def assert_cycles_are_the_variables(circ):
    perm = wiring_permutation(circ.wire_vars)
    assert cycles(perm) == position_sets(circ.wire_vars)
    return perm


def test_end_bit_rule():
    assert ws.END_BIT_MIN == 33
    assert [ws.end_bit(nv) for nv in (1, 2, 3, 4, 5, 256, 257)] == [33, 33, 34, 34, 35, 40, 41]
    for b in range(1, 33):  # num_vars - 1 of exactly b bits needs them all, one bit fewer does not
        assert ws.end_bit((1 << (b - 1)) + 1) == 32 + b
        assert ws.end_bit(1 << b) == 32 + b
    assert ws.end_bit((1 << 32) - 1) == 64 and ws.end_bit((1 << 31) + 1) == 64 and ws.end_bit((1 << 24) + 1) == 57
    assert ws.CYCLE_THREADS == 256


@pytest.mark.parametrize("num_vars", ws.INDEX_WIDTHS)
def test_index_width_shape(num_vars):
    s = ws.index_width(num_vars)
    circ, wv = s.circ, s.circ.wire_vars.reshape(-1)
    assert s.num_vars == num_vars and f"end_bit {ws.end_bit(num_vars)}" in s.claim
    assert int(wv.min()) == 0 and int(wv.max()) == num_vars - 1
    assert set(s.values) == set(np.unique(wv).tolist())
    b = ws.index_bits(num_vars)
    if num_vars == 1:
        assert s.top_pairs == [] and (wv == 0).all()
    else:
        assert b == (num_vars - 1).bit_length() and s.top_pairs
        for v, w in s.top_pairs:  # equal below the top index bit the sort reads, different in it
            assert w - v == 1 << (b - 1) and v >> (b - 1) == 0 and w >> (b - 1) == 1 and w < num_vars
            assert any(wv[p] == v and wv[p + 1] == w for p in range(len(wv) - 1)), (v, w)
        # a sort one bit short sees each pair as one variable: other cycles
        short = wv & np.uint32((1 << (b - 1)) - 1)
        assert cycles(wiring_permutation(short)) != cycles(wiring_permutation(wv))
    assert_cycles_are_the_variables(circ)
    if circ.witness is None:
        assert num_vars > ws.MAX_WITNESS_VARS
    else:
        assert circ.witness.shape == (num_vars, 4)
        assert (expand(circ)[0, 0] == synth.to_mont_array([s.values[int(wv[0])]])[0]).all()


@pytest.mark.parametrize("log_n", [6, 16, 17])
def test_cycle_shapes(log_n):
    n = 1 << log_n
    s = ws.one_variable(log_n)
    assert cycles(wiring_permutation(s.circ.wire_vars)) == {frozenset(range(5 * n))}
    s = ws.each_once_descending(log_n)
    assert (wiring_permutation(s.circ.wire_vars) == np.arange(5 * n)).all() and s.num_vars == 5 * n
    assert int(s.circ.wire_vars[0, 0]) == 5 * n - 1
    s = ws.block_boundary_pairs(log_n)
    wv = s.circ.wire_vars.reshape(-1)
    sv = np.sort(wv)  # the sorted keys' variables, in sorted order
    counts = np.bincount(wv)
    for t in range(ws.CYCLE_THREADS, 5 * n, ws.CYCLE_THREADS):
        assert sv[t - 1] == sv[t] and counts[sv[t]] == 2, t
    assert_cycles_are_the_variables(s.circ)
    s = ws.stride_n(log_n)
    assert cycles(wiring_permutation(s.circ.wire_vars)) == {frozenset(range(j, 5 * n, n)) for j in range(n)}
    for s in (ws.one_variable(log_n), ws.each_once_descending(log_n), ws.stride_n(log_n)):
        assert not s.circ.selectors.any() and s.circ.num_inputs == 0
        assert (expand(s.circ) == s.circ.witness[s.circ.wire_vars]).all()


@pytest.mark.parametrize("log_n", [4, 10, 13])
def test_dense_shape(log_n):
    s = ws.dense(log_n)
    assert_cycles_are_the_variables(s.circ)
    assert_gates_and_public_inputs(s.circ)


@pytest.mark.parametrize("log_n,num_inputs,shared,zero", [
    (6, 0, False, False), (6, 1, False, False), (6, 5, True, True), (10, 9, True, True), (13, 4097, False, False),
    (13, 4097, True, True)])
def test_public_input_shapes(log_n, num_inputs, shared, zero):
    s = ws.public_inputs(log_n, num_inputs, shared=shared, zero=zero)
    circ = s.circ
    assert circ.num_inputs == num_inputs == circ.pub_inputs.shape[0]
    if shared:
        assert circ.wire_vars[4, 1] == circ.wire_vars[4, num_inputs - 1]
        assert (circ.pub_inputs[1] == circ.pub_inputs[num_inputs - 1]).all()
    if zero:
        assert circ.wire_vars[4, 0] == 0 and not circ.pub_inputs[0].any()
    assert_cycles_are_the_variables(circ)
    assert_gates_and_public_inputs(circ)


@pytest.mark.parametrize("log_n", [5, 10])
def test_every_row_public(log_n):
    n = 1 << log_n
    circ = ws.every_row_public(log_n).circ
    assert circ.num_inputs == n and circ.pub_inputs.shape == (n, 4)
    assert circ.wire_vars[4, 0] == 0 and circ.wire_vars[4, 1] == circ.wire_vars[4, n - 1]
    assert not circ.pub_inputs[0].any() and (circ.pub_inputs[1] == circ.pub_inputs[n - 1]).all()
    assert_cycles_are_the_variables(circ)
    assert_gates_and_public_inputs(circ)


@pytest.mark.parametrize("log_n", [5, 10])
def test_unused_variables(log_n):
    n = 1 << log_n
    s = ws.unused_variables(log_n)
    circ = s.circ
    # longer than the NTT scratch a context holds after preprocessing and proving any key of this domain size
    assert s.num_vars == 128 * n == circ.num_vars and s.num_vars > ws.staging_floor(log_n)
    used = np.unique(circ.wire_vars)
    assert int(used.max()) == s.num_vars - 1 and len(used) < s.num_vars // 10
    assert_cycles_are_the_variables(circ)
    assert_gates_and_public_inputs(circ)


def test_staging_floor():
    """NS * m from preprocess is the larger of the two reservations at every domain size: 78n from 2^4 on, 104n below."""
    assert (ws.NS, ws.STAGE_PER_M, ws.COSET_SWITCH, ws.COSETS_LARGE, ws.COSETS_SMALL) == (13, 7, 4, 6, 8)
    assert [ws.staging_floor(log_n) >> log_n for log_n in (2, 3, 4, 10, 17)] == [104, 104, 78, 78, 78]


@pytest.mark.parametrize("log_n", [5, 8])
def test_dense_witnesses_are_distinct_and_satisfying(log_n):
    circ = ws.dense(log_n, num_inputs=2, seed=0x65 + log_n).circ
    variants = ws.dense_witnesses(circ, 4, seed=log_n)
    for i, w in enumerate(variants):
        other = ws.with_witness(circ, w)
        assert_gates_and_public_inputs(other)
        assert w.shape == circ.witness.shape and not w[0].any()
        assert not (w == circ.witness).all() and all(not (w == u).all() for u in variants[:i])
        assert (expand(other) == w[circ.wire_vars]).all()


SMALL = [
    lambda: ws.one_variable(6), lambda: ws.each_once_descending(6), lambda: ws.block_boundary_pairs(6),
    lambda: ws.stride_n(6), lambda: ws.dense(6, num_inputs=3), lambda: ws.public_inputs(6, 5, shared=True, zero=True),
    lambda: ws.every_row_public(5), lambda: ws.unused_variables(5), lambda: ws.index_width(257),
    lambda: ws.index_width((1 << 16) + 1), lambda: ws.index_width(1),
]


@pytest.mark.parametrize("build", SMALL, ids=["one_variable", "each_once", "block_boundary", "stride_n", "dense",
                                              "public_shared_zero", "every_row_public", "unused", "index_257",
                                              "index_65537", "index_1"])
def test_oracle_proves_small_shapes(oracle, pyoracle, build):
    py = pyoracle
    circ = build().circ
    log_n = circ.log_n
    assert circ.n <= 1 << 6
    tau = py.to_mont(0xB200B201 % py.R, py.R)
    tau = oracle.int_to_limbs(tau)
    srs = oracle.srs_from_tau(tau, circ.n + 3)
    opk = oracle.plonk_preprocess(log_n, circ.selectors, wiring_permutation(circ.wire_vars), circ.k, srs)
    wires = np.ascontiguousarray(expand(circ))
    pub = np.ascontiguousarray(circ.witness[circ.wire_vars[4, :circ.num_inputs]]).reshape(-1, 4)
    rc, proof, _, _ = oracle.plonk_prove(log_n, circ.num_inputs, circ.k, opk, wires, pub, synth.splitmix_blinders(11), srs)
    assert rc == 0
    assert oracle.plonk_verify_known_tau(log_n, circ.num_inputs, circ.k, opk, pub, proof, tau)
