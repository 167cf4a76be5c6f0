"""Proving from the witness vector (`b200_plonk_preprocess_wiring`, `b200_plonk_prove_witness`, `_witness_batch`,
`b200_pool_submit_prove_witness`): a key made from the circuit's wiring is the key `b200_plonk_preprocess` makes from
the permutation the wiring implies, and a proof made from the witness vector is, byte for byte, the proof
`b200_plonk_prove` makes from the expanded 5 x n table — eagerly and from replayed graphs, from host and device
pointers, alone, in a batch and through the pool.  Every bad input is refused with an error code."""
import ctypes as C
import random

import numpy as np
import pytest

from renegade_b200 import _lib, synth
from renegade_b200.backend import B200WitnessItem, PlonkKzgSnark, ProverPool, VerifyingKey
from test_prove_witness_cpu import expand, wiring_permutation

pytestmark = pytest.mark.gpu

TAU = 0x1D2C3B4A59687706F5E4D3C2B1A09F8E7D6C5B4A39281706F5E4D3C2B1A0987  # conftest's SRS_2_16_TAU: srs_2_16_g2 is its G2 pair
INVALID, UNSAT = -1, -7


def load_srs(ctx, oracle, pyoracle, n):
    tau = oracle.int_to_limbs(pyoracle.to_mont(TAU % pyoracle.R, pyoracle.R))
    return ctx.load_bases(oracle.srs_from_tau(tau, n + 3))


def keys(ctx, bases, circ):
    """(key from the wiring, key from the permutation the wiring implies)"""
    wpk = PlonkKzgSnark.preprocess_wiring(ctx, bases, circ.log_n, circ.num_inputs, circ.selectors, circ.wire_vars,
                                          circ.num_vars, circ.k)
    pk = PlonkKzgSnark.preprocess(ctx, bases, circ.log_n, circ.num_inputs, circ.selectors,
                                  wiring_permutation(circ.wire_vars), circ.k)
    return wpk, pk


def from_table(ctx, pk, circ, bl):
    proof, hint, ch = PlonkKzgSnark.prove_with_link_hint(ctx, pk, expand(circ), circ.pub_inputs, bl, want_challenges=True)
    return bytes(proof), hint.linking_wire_poly.tobytes(), ch.tobytes()


def from_witness(ctx, pk, witness, bl):
    proof, hint, pub, ch = PlonkKzgSnark.prove_witness(ctx, pk, witness, bl, want_challenges=True)
    return (bytes(proof), hint.linking_wire_poly.tobytes(), ch.tobytes()), pub


@pytest.mark.parametrize("log_n,link", [(4, False), (4, True), (10, False), (10, True), (13, False), (13, True)])
def test_key_from_wiring_is_the_key_from_its_permutation(ctx, oracle, pyoracle, log_n, link):
    lk = (log_n - 1, 2, [11, 12, 13]) if link else None
    circ = synth.synth_circuit(log_n, num_inputs=2, seed=300 + log_n, link=lk)
    bases = load_srs(ctx, oracle, pyoracle, circ.n)
    wpk, pk = keys(ctx, bases, circ)
    assert (wpk.selector_comms == pk.selector_comms).all() and (wpk.sigma_comms == pk.sigma_comms).all()
    assert wpk.num_vars == circ.num_vars and pk.num_vars == 0
    # a different walk of the same cycles (SynthCircuit.perm) is another key
    other = PlonkKzgSnark.preprocess(ctx, bases, log_n, circ.num_inputs, circ.selectors, circ.perm, circ.k)
    assert (other.selector_comms == pk.selector_comms).all() and not (other.sigma_comms == pk.sigma_comms).all()
    for k in (wpk, pk, other):
        k.free()
    bases.free()


def test_restated_statement_key_and_proof(ctx, oracle, pyoracle):
    from host_circuits import valid_balance_create as vbc
    witness, statement = vbc.create_witness_statement(seed=0xB200)
    circ = vbc.ValidBalanceCreate.build(witness, statement).finalize_for_arithmetization()
    assert circ.log_n == 13 and circ.num_inputs == 13 and circ.num_vars < 2 * circ.n
    bases = load_srs(ctx, oracle, pyoracle, circ.n)
    wpk, pk = keys(ctx, bases, circ)
    assert (wpk.selector_comms == pk.selector_comms).all() and (wpk.sigma_comms == pk.sigma_comms).all()
    bl = synth.splitmix_blinders(0x77)
    got, pub = from_witness(ctx, wpk, circ.witness, bl)
    assert got == from_table(ctx, pk, circ, bl)
    assert (pub == synth.to_mont_array(statement.to_scalars())).all()
    wpk.free()
    pk.free()
    bases.free()


def test_proof_identity_eager_replayed_host_and_device(ctx, oracle, pyoracle, srs_2_16_g2):
    import torch
    circ = synth.synth_circuit(11, num_inputs=3, seed=71, link=(9, 4, [1, 2, 3, 4]))
    bases = load_srs(ctx, oracle, pyoracle, circ.n)
    wpk, pk = keys(ctx, bases, circ)
    ctx.use_graphs(True)
    bls = [synth.splitmix_blinders(500 + i) for i in range(6)]
    want = [from_table(ctx, pk, circ, b) for b in bls]
    wit = np.ascontiguousarray(circ.witness)
    d_w = torch.from_numpy(wit.view(np.int64)).cuda()
    h_w = torch.from_numpy(wit.view(np.int64)).pin_memory()
    torch.cuda.synchronize()
    g0 = ctx.graph_launches()
    sources = [wit, wit, wit, d_w.data_ptr(), h_w.data_ptr(), d_w.data_ptr()]  # 1st eager, 2nd captured, 3rd on replayed
    for i, (src, bl) in enumerate(zip(sources, bls)):
        got, pub = from_witness(ctx, wpk, src, bl)
        assert got == want[i], i
        assert (pub == circ.pub_inputs).all(), i
    assert ctx.graph_launches() - g0 == 5 * 7  # every proof after the first ran as 7 graph submissions
    # the table path of the same key gives the same bytes too, and the verifier accepts
    assert from_table(ctx, wpk, circ, bls[0]) == want[0]
    proof = PlonkKzgSnark.prove_witness(ctx, wpk, wit, bls[0])[0]
    vk = VerifyingKey.from_proving_key(wpk, *srs_2_16_g2)
    assert PlonkKzgSnark.verify(vk, circ.pub_inputs, proof)
    wrong = circ.pub_inputs.copy()
    wrong[0, 0] ^= 1
    assert not PlonkKzgSnark.verify(vk, wrong, proof)
    wpk.free()
    pk.free()
    bases.free()


def unsatisfying(circ):
    """A witness vector that breaks one gate: the output variable of a gate past the public inputs takes another value."""
    bad = circ.witness.copy()
    v = int(circ.wire_vars[4, circ.num_inputs + 3])
    bad[v] = bad[int(circ.wire_vars[4, circ.num_inputs + 4])]
    return bad


def test_batch_items_equal_single_proofs(ctx, oracle, pyoracle, monkeypatch):
    import torch
    circ = synth.synth_circuit(8, num_inputs=2, seed=8)
    bases = load_srs(ctx, oracle, pyoracle, circ.n)
    wpk, pk = keys(ctx, bases, circ)
    bls = [synth.splitmix_blinders(300 + i) for i in range(7)]
    want = [from_table(ctx, pk, circ, b) for b in bls]
    zero = bytes(len(want[0][0]))
    bad = unsatisfying(circ)
    d_w = torch.from_numpy(np.ascontiguousarray(circ.witness).view(np.int64)).cuda()
    torch.cuda.synchronize()

    def batch(witnesses):
        proofs, hints, st, pubs, chs = PlonkKzgSnark.prove_witness_batch(ctx, wpk, witnesses, bls[:len(witnesses)],
                                                                         link_hints=True, want_challenges=True)
        return [(bytes(p), h.linking_wire_poly.tobytes() if h is not None else None, c.tobytes())
                for p, h, c in zip(proofs, hints, chs)], st, pubs

    for k in (1, 2, 7):
        got, st, pubs = batch([circ.witness] * k)
        assert st == [0] * k and got == want[:k]
        assert all((p == circ.pub_inputs).all() for p in pubs)
    mixed = [circ.witness, bad, d_w.data_ptr(), circ.witness, d_w.data_ptr(), bad, circ.witness]
    one, st1, _ = batch(mixed)
    assert st1 == [0, UNSAT, 0, 0, 0, UNSAT, 0]
    for i in range(7):
        if st1[i]:
            assert one[i][0] == zero and one[i][1] is None
        else:
            assert one[i] == want[i], i
    for chunk in ("1", "3"):
        monkeypatch.setenv("B200_PROVE_BATCH_CHUNK", chunk)
        got, st, _ = batch(mixed)
        assert st == st1 and got == one, chunk
    monkeypatch.delenv("B200_PROVE_BATCH_CHUNK")
    with pytest.raises(_lib.B200Error) as err:  # alone, an unsatisfying witness is the call's error
        PlonkKzgSnark.prove_witness(ctx, wpk, bad, bls[0])
    assert err.value.code == UNSAT
    assert from_witness(ctx, wpk, circ.witness, bls[0])[0] == want[0]  # the context keeps proving
    wpk.free()
    pk.free()
    bases.free()


def test_pool_jobs_equal_single_proofs(ctx, oracle, pyoracle):
    circ = synth.synth_circuit(9, num_inputs=2, seed=55)
    bases = load_srs(ctx, oracle, pyoracle, circ.n)
    wpk0, pk0 = keys(ctx, bases, circ)
    bls = [synth.splitmix_blinders(1200 + i) for i in range(32)]
    want = [from_table(ctx, pk0, circ, b)[:2] for b in bls]
    wpk0.free()
    pk0.free()
    bases.free()
    pool = ProverPool(device=0, workers=4)
    try:
        pc = pool.context(0)
        b2 = load_srs(pc, oracle, pyoracle, circ.n)
        wpk = PlonkKzgSnark.preprocess_wiring(pc, b2, circ.log_n, circ.num_inputs, circ.selectors, circ.wire_vars,
                                              circ.num_vars, circ.k)
        wires = np.ascontiguousarray(expand(circ))
        tickets = []
        for i, bl in enumerate(bls):  # witness jobs interleaved with ordinary jobs on the same key
            tickets.append(pool.submit_prove_witness(wpk, circ.witness, bl, with_link_poly=True))
            if i % 4 == 0:
                tickets.append(pool.submit_prove(wpk, wires.ctypes.data, circ.pub_inputs, bl, with_link_poly=True, keep=wires))
        results = [pool.wait(t) for t in tickets]
        it = iter(results)
        for i in range(32):
            proof, link, pub = next(it)
            assert (bytes(proof), link.tobytes()) == want[i], i
            assert (pub == circ.pub_inputs).all()
            if i % 4 == 0:
                proof, link = next(it)
                assert (bytes(proof), link.tobytes()) == want[i], i
        with pytest.raises(_lib.B200Error) as err:
            pool.wait(pool.submit_prove_witness(wpk, unsatisfying(circ), bls[0]))
        assert err.value.code == UNSAT
        pk = PlonkKzgSnark.preprocess(pc, b2, circ.log_n, circ.num_inputs, circ.selectors, circ.perm, circ.k)
        with pytest.raises(_lib.B200Error) as err:  # a key without wiring is refused at submit
            pool.submit_prove_witness(pk, wires.ctypes.data, bls[0])
        assert err.value.code == INVALID and "wiring" in str(err.value)
        pk.free()
        wpk.free()
        b2.free()
    finally:
        pool.close()


def tiny(log_n, wire_vars, witness_ints, num_inputs=0):
    """A circuit without gate constraints (all selectors zero) over a given wiring: any witness satisfies it."""
    n = 1 << log_n
    return synth.SynthCircuit(
        log_n=log_n, num_inputs=num_inputs, k=synth.to_mont_array([pow(5, i, synth.R) for i in range(5)]),
        selectors=np.zeros((13, n, 4), dtype=np.uint64), perm=None, wires=None, pub_inputs=None, n_gates=n,
        selectors_int=None, wires_int=None, pub_inputs_int=None,
        wire_vars=np.asarray(wire_vars, dtype=np.uint32).reshape(5, n), witness=synth.to_mont_array(witness_ints))


@pytest.mark.parametrize("case", ["one_variable", "each_once", "unused_numbers", "num_vars_1"])
def test_wiring_edges(ctx, oracle, pyoracle, case):
    log_n, n = 4, 16
    rnd = random.Random(9)
    if case in ("one_variable", "num_vars_1"):  # every position the same variable
        nv = 1 if case == "num_vars_1" else 3
        wv = np.full(5 * n, nv - 1, dtype=np.uint32)
    elif case == "each_once":                  # every variable used exactly once, in descending order
        nv, wv = 5 * n, np.arange(5 * n, dtype=np.uint32)[::-1].copy()
    else:                                        # only multiples of 7 below 1000 are used
        nv, wv = 1000, np.array([7 * rnd.randrange(100) for _ in range(5 * n)], dtype=np.uint32)
    circ = tiny(log_n, wv, [rnd.randrange(synth.R) for _ in range(nv)])
    bases = load_srs(ctx, oracle, pyoracle, n)
    wpk, pk = keys(ctx, bases, circ)
    assert (wpk.sigma_comms == pk.sigma_comms).all() and wpk.num_vars == nv and wpk.num_inputs == 0
    bl = synth.splitmix_blinders(4)
    proof, hint, ch = PlonkKzgSnark.prove_with_link_hint(ctx, pk, expand(circ), np.zeros((0, 4), dtype=np.uint64), bl,
                                                         want_challenges=True)
    got, pub = from_witness(ctx, wpk, circ.witness, bl)
    assert got == (bytes(proof), hint.linking_wire_poly.tobytes(), ch.tobytes()) and pub.shape == (0, 4)
    wpk.free()
    pk.free()
    bases.free()


def test_bad_arguments(ctx, oracle, pyoracle):
    circ = synth.synth_circuit(5, num_inputs=2, seed=3)
    bases = load_srs(ctx, oracle, pyoracle, circ.n)
    lib = ctx._lib
    bl = synth.splitmix_blinders(1)
    # an index == num_vars: refused, the message names the first such position, and the context still works
    wv = circ.wire_vars.copy().reshape(-1)
    wv[37] = circ.num_vars
    wv[101] = circ.num_vars + 5
    with pytest.raises(_lib.B200Error) as err:
        PlonkKzgSnark.preprocess_wiring(ctx, bases, circ.log_n, circ.num_inputs, circ.selectors, wv, circ.num_vars, circ.k)
    assert err.value.code == INVALID and "wire_vars[37]" in str(err.value)
    with pytest.raises(_lib.B200Error) as err:
        PlonkKzgSnark.preprocess_wiring(ctx, bases, circ.log_n, circ.num_inputs, circ.selectors, circ.wire_vars, 0, circ.k)
    assert err.value.code == INVALID
    wpk, pk = keys(ctx, bases, circ)
    want = from_table(ctx, pk, circ, bl)
    assert from_witness(ctx, wpk, circ.witness, bl)[0] == want
    # a key made by b200_plonk_preprocess holds no wiring
    proof = (C.c_uint64 * 144)()
    wit = np.ascontiguousarray(circ.witness)
    p = lambda a: a.ctypes.data_as(C.c_void_p)  # noqa: E731
    assert lib.b200_plonk_prove_witness(ctx._h, pk._h, p(wit), p(bl), proof, None, None, None) == INVALID
    assert b"wiring" in lib.b200_last_error()
    st = (C.c_int * 1)()
    items = (B200WitnessItem * 1)()
    items[0] = B200WitnessItem(p(wit), p(bl), C.cast(proof, C.c_void_p), None, None, None)
    assert lib.b200_plonk_prove_witness_batch(ctx._h, pk._h, items, 1, st) == INVALID
    # NULL pointers
    assert lib.b200_plonk_prove_witness(ctx._h, wpk._h, None, p(bl), proof, None, None, None) == INVALID
    assert lib.b200_plonk_prove_witness(ctx._h, wpk._h, p(wit), None, proof, None, None, None) == INVALID
    assert lib.b200_plonk_prove_witness(ctx._h, wpk._h, p(wit), p(bl), None, None, None, None) == INVALID
    assert lib.b200_plonk_prove_witness(None, wpk._h, p(wit), p(bl), proof, None, None, None) == INVALID
    assert lib.b200_plonk_prove_witness_batch(ctx._h, wpk._h, None, 0, st) == 0
    assert lib.b200_plonk_prove_witness_batch(ctx._h, wpk._h, None, 1, st) == INVALID
    items[0] = B200WitnessItem(None, p(bl), C.cast(proof, C.c_void_p), None, None, None)
    assert lib.b200_plonk_prove_witness_batch(ctx._h, wpk._h, items, 1, st) == INVALID
    assert b"item 0" in lib.b200_last_error()
    h = C.c_void_p()
    sel = np.ascontiguousarray(circ.selectors)
    assert lib.b200_plonk_preprocess_wiring(ctx._h, bases._h, 5, 2, p(sel), None, circ.num_vars, p(circ.k), C.byref(h)) == INVALID
    with pytest.raises(ValueError):
        PlonkKzgSnark.prove_witness(ctx, wpk, wit[:-1], bl)
    assert lib.b200_plonk_prove_witness(ctx._h, wpk._h, p(wit), p(bl), proof, None, None, None) == 0
    assert bytes(proof) == want[0]
    wpk.free()
    pk.free()
    bases.free()


def test_launch_accounting(ctx, oracle, pyoracle):
    circ = synth.synth_circuit(11, num_inputs=3, seed=44)
    bases = load_srs(ctx, oracle, pyoracle, circ.n)
    wpk, _pk = keys(ctx, bases, circ)
    _pk.free()
    ctx.use_graphs(True)
    bls = [synth.splitmix_blinders(60 + i) for i in range(4)]
    for on in (False, True):  # eager, then replayed graphs
        ctx.use_graphs(on)
        for b in bls[:2]:
            from_table(ctx, wpk, circ, b)
        k0, g0 = ctx.kernel_launches(), ctx.graph_launches()
        a = from_table(ctx, wpk, circ, bls[2])
        k1, g1 = ctx.kernel_launches(), ctx.graph_launches()
        b = from_witness(ctx, wpk, circ.witness, bls[2])[0]
        k2, g2 = ctx.kernel_launches(), ctx.graph_launches()
        assert a == b
        assert k2 - k1 == (k1 - k0) + 1          # the gather is one launch
        assert g2 - g1 == g1 - g0 == (7 if on else 0)
    ctx.use_graphs(True)
    wpk.free()
    bases.free()


def test_circuit_types_opt_in(ctx, srs_2_16, srs_2_16_g2):
    import renegade_b200 as rb
    from host_circuits import statements as st
    from host_circuits import valid_balance_create as vbc
    from renegade_b200 import circuit_types as ct

    class FromWitness(st.ValidBalanceCreate):
        prove_from_witness = True

        @classmethod
        def name(cls):
            return "Valid Balance Create (from the witness vector)"

    params = rb.parse_ptau_file(ctx, srs_2_16, count=(1 << 16) + 3)
    ct.set_system_srs(ctx, params.powers_of_g, *srs_2_16_g2)
    try:
        insts = [vbc.create_witness_statement(seed) for seed in (3, 4)]
        assert FromWitness.proving_key().num_vars > 0 and st.ValidBalanceCreate.proving_key().num_vars == 0
        for w, s in insts:
            proof, hint = ct.singleprover_prove_with_hint(FromWitness, w, s, rng=random.Random(1))
            ct.verify_singleprover_proof(FromWitness, s, proof)
            assert hint.linking_wire_poly.shape == (FromWitness.proving_key().domain_size + 2, 4)
        got = ct.singleprover_prove_batch(FromWitness, insts, rng=random.Random(2))
        rng = random.Random(2)
        for (w, s), proof in zip(insts, got):
            assert bytes(proof) == bytes(ct.singleprover_prove(FromWitness, w, s, rng=rng))
        with pytest.raises(ct.ProverError):
            ct.singleprover_prove(FromWitness, vbc.create_witness_statement(9)[0], insts[0][1])
    finally:
        ct.clear_key_cache()
