"""Batch proving (`b200_plonk_prove_batch`, `PlonkKzgSnark.prove_batch`, `ProverPool.submit_prove_batch`,
`circuit_types.singleprover_prove_batch`): k witnesses of one key proved by one call must give, item by item, the bytes
`b200_plonk_prove` gives for the same witness and blinders — proof, link polynomial and challenges — whatever the
chunking, the pointer kinds and the unsatisfied items around them, and without disturbing the single prover's graphs."""
import ctypes as C
import random
import threading

import numpy as np
import pytest

from renegade_b200 import synth
from renegade_b200.backend import PlonkKzgSnark, ProverPool

pytestmark = pytest.mark.gpu

TAU = 0x1D2C3B4A59687706F5E4D3C2B1A09F8E7D6C5B4A39281706F5E4D3C2B1A0987  # conftest's SRS_2_16_TAU: srs_2_16_g2 is its G2 pair
UNSAT = -7


def make(ctx, oracle, pyoracle, log_n, num_inputs, seed):
    circ = synth.synth_circuit(log_n, num_inputs=num_inputs, seed=seed, check=(log_n <= 10))
    tau = oracle.int_to_limbs(pyoracle.to_mont(TAU % pyoracle.R, pyoracle.R))
    srs = oracle.srs_from_tau(tau, (1 << log_n) + 3)
    bases = ctx.load_bases(srs)
    pk = PlonkKzgSnark.preprocess(ctx, bases, log_n, circ.num_inputs, circ.selectors, circ.perm, circ.k)
    return circ, srs, bases, pk


def single(ctx, pk, wires, pub_inputs, bl):
    proof, hint, ch = PlonkKzgSnark.prove_with_link_hint(ctx, pk, wires, pub_inputs, bl, want_challenges=True)
    return bytes(proof), hint.linking_wire_poly.tobytes(), ch.tobytes()


def batch(ctx, pk, wires, pis, bls):
    proofs, hints, st, chs = PlonkKzgSnark.prove_batch(ctx, pk, wires, pis, bls, link_hints=True, want_challenges=True)
    out = [(bytes(p), h.linking_wire_poly.tobytes() if h is not None else None, c.tobytes()) for p, h, c in zip(proofs, hints, chs)]
    return out, st


def unsatisfied(circ):
    bad = circ.wires.copy()
    bad[4, circ.num_inputs + 3] = bad[4, circ.num_inputs + 4]
    return bad


# n = 16 and 256: a segment of the grand-product scan is exactly one chunk / exactly 16 chunks
@pytest.mark.parametrize("log_n,num_inputs", [(2, 0), (3, 2), (4, 1), (5, 2), (8, 3), (10, 0), (10, 5), (12, 2), (13, 4)])
def test_batch_equals_single_proofs(ctx, oracle, pyoracle, log_n, num_inputs):
    circ, srs, bases, pk = make(ctx, oracle, pyoracle, log_n, num_inputs, seed=11 + log_n)
    bls = [synth.splitmix_blinders(7000 + 31 * i + log_n) for i in range(17)]
    want = [single(ctx, pk, circ.wires, circ.pub_inputs, b) for b in bls]
    for k in (1, 2, 3, 17):
        got, st = batch(ctx, pk, [circ.wires] * k, [circ.pub_inputs] * k, bls[:k])
        assert st == [0] * k
        assert got == want[:k], (log_n, num_inputs, k)
    if log_n == 3:  # and the CPU oracle prover
        for i in range(3):
            rc, oproof, och, olink = oracle.plonk_prove(log_n, circ.num_inputs, circ.k, oracle.plonk_preprocess(
                log_n, circ.selectors, circ.perm, circ.k, srs), circ.wires, circ.pub_inputs, bls[i], srs, True)
            assert rc == 0 and bytes(oproof) == want[i][0]
            assert np.ascontiguousarray(olink, dtype=np.uint64).tobytes() == want[i][1]
            assert bytes(och) == want[i][2]
    pk.free()
    bases.free()


def test_duplicates(ctx, oracle, pyoracle, srs_2_16_g2):
    circ, srs, bases, pk = make(ctx, oracle, pyoracle, 7, 3, seed=5)
    b0, b1 = synth.splitmix_blinders(1), synth.splitmix_blinders(2)
    got, st = batch(ctx, pk, [circ.wires] * 3, [circ.pub_inputs] * 3, [b0, b0, b1])
    assert st == [0, 0, 0]
    assert got[0] == got[1] and got[0][0] != got[2][0]
    from renegade_b200.backend import VerifyingKey
    proofs, _, _ = PlonkKzgSnark.prove_batch(ctx, pk, [circ.wires] * 2, [circ.pub_inputs] * 2, [b0, b1])
    vk = VerifyingKey.from_proving_key(pk, *srs_2_16_g2)
    assert all(PlonkKzgSnark.verify(vk, circ.pub_inputs, p) for p in proofs)
    pk.free()
    bases.free()


def test_unsatisfied_items(ctx, oracle, pyoracle):
    circ, srs, bases, pk = make(ctx, oracle, pyoracle, 6, 2, seed=8)
    bad = unsatisfied(circ)
    bls = [synth.splitmix_blinders(300 + i) for i in range(5)]
    want = [single(ctx, pk, circ.wires, circ.pub_inputs, b) for b in bls]
    zero = bytes(len(want[0][0]))
    for bad_at in ([0], [2], [4], [0, 2, 4]):
        wires = [bad if i in bad_at else circ.wires for i in range(5)]
        got, st = batch(ctx, pk, wires, [circ.pub_inputs] * 5, bls)
        assert st == [UNSAT if i in bad_at else 0 for i in range(5)], bad_at
        for i in range(5):
            if i in bad_at:
                assert got[i][0] == zero and got[i][1] is None
            else:
                assert got[i] == want[i], (bad_at, i)
    got, st = batch(ctx, pk, [bad] * 3, [circ.pub_inputs] * 3, bls[:3])
    assert st == [UNSAT] * 3 and all(g[0] == zero for g in got)
    assert single(ctx, pk, circ.wires, circ.pub_inputs, bls[0]) == want[0]  # the context keeps proving
    pk.free()
    bases.free()


def test_host_and_device_wire_pointers(ctx, oracle, pyoracle):
    import torch
    circ, srs, bases, pk = make(ctx, oracle, pyoracle, 9, 1, seed=21)
    bls = [synth.splitmix_blinders(40 + i) for i in range(4)]
    want = [single(ctx, pk, circ.wires, circ.pub_inputs, b) for b in bls]
    d_w = torch.from_numpy(np.ascontiguousarray(circ.wires).view(np.int64)).cuda()
    h_w = torch.from_numpy(np.ascontiguousarray(circ.wires).view(np.int64)).pin_memory()
    torch.cuda.synchronize()
    wires = [d_w.data_ptr(), circ.wires, h_w.data_ptr(), d_w.data_ptr()]
    got, st = batch(ctx, pk, wires, [circ.pub_inputs] * 4, bls)
    assert st == [0] * 4 and got == want
    pk.free()
    bases.free()


def test_chunking_does_not_change_the_bytes(ctx, oracle, pyoracle, monkeypatch):
    circ, srs, bases, pk = make(ctx, oracle, pyoracle, 8, 2, seed=33)
    bad = unsatisfied(circ)
    bls = [synth.splitmix_blinders(900 + i) for i in range(7)]
    wires = [bad if i in (1, 5) else circ.wires for i in range(7)]
    one, st1 = batch(ctx, pk, wires, [circ.pub_inputs] * 7, bls)
    for chunk in ("1", "2", "3"):
        monkeypatch.setenv("B200_PROVE_BATCH_CHUNK", chunk)
        got, st = batch(ctx, pk, wires, [circ.pub_inputs] * 7, bls)
        assert st == st1 and got == one, chunk
    monkeypatch.delenv("B200_PROVE_BATCH_CHUNK")
    assert st1 == [0, UNSAT, 0, 0, 0, UNSAT, 0]
    pk.free()
    bases.free()


def test_single_proofs_keep_their_graphs(ctx, oracle, pyoracle):
    circ, srs, bases, pk = make(ctx, oracle, pyoracle, 11, 3, seed=44)
    ctx.use_graphs(True)
    bls = [synth.splitmix_blinders(60 + i) for i in range(6)]
    single(ctx, pk, circ.wires, circ.pub_inputs, bls[0])  # eager
    single(ctx, pk, circ.wires, circ.pub_inputs, bls[1])  # captured
    k0, g0 = ctx.kernel_launches(), ctx.graph_launches()
    before = [single(ctx, pk, circ.wires, circ.pub_inputs, b) for b in bls[2:4]]
    per_proof, kernels = (ctx.graph_launches() - g0) / 2, ctx.kernel_launches() - k0
    g1 = ctx.graph_launches()
    got, st = batch(ctx, pk, [circ.wires] * 4, [circ.pub_inputs] * 4, bls[2:6])
    assert ctx.graph_launches() == g1  # a batch runs eagerly
    k0, g2 = ctx.kernel_launches(), ctx.graph_launches()
    after = [single(ctx, pk, circ.wires, circ.pub_inputs, b) for b in bls[2:4]]
    assert (ctx.graph_launches() - g2) / 2 == per_proof == 7
    assert ctx.kernel_launches() - k0 == kernels  # the same kernels, submitted as the same 7 graphs per proof
    assert after == before == got[:2]
    pk.free()
    bases.free()


def test_pool_batches_from_two_threads(ctx, oracle, pyoracle):
    circ, srs, bases, pk0 = make(ctx, oracle, pyoracle, 9, 2, seed=55)
    bls = [synth.splitmix_blinders(1200 + i) for i in range(12)]
    want = [single(ctx, pk0, circ.wires, circ.pub_inputs, b)[0] for b in bls]
    pk0.free()
    bases.free()
    pool = ProverPool(device=0, workers=2)
    try:
        pc = pool.context(0)
        b2 = pc.load_bases(srs)
        pk = PlonkKzgSnark.preprocess(pc, b2, 9, circ.num_inputs, circ.selectors, circ.perm, circ.k)
        results = {}

        def worker(t):
            idx = list(range(6 * t, 6 * t + 6))
            tb = pool.submit_prove_batch(pk, [circ.wires] * 3, [circ.pub_inputs] * 3, [bls[i] for i in idx[:3]])
            wires = np.ascontiguousarray(circ.wires)
            ts = pool.submit_prove(pk, wires.ctypes.data, circ.pub_inputs, bls[idx[3]], keep=wires)
            tb2 = pool.submit_prove_batch(pk, [circ.wires] * 2, [circ.pub_inputs] * 2, [bls[i] for i in idx[4:]])
            p, _, st = pool.wait(tb)
            assert st == [0, 0, 0]
            results.update({i: bytes(x) for i, x in zip(idx[:3], p)})
            results[idx[3]] = bytes(pool.wait(ts))
            p, _, st = pool.wait(tb2)
            assert st == [0, 0]
            results.update({i: bytes(x) for i, x in zip(idx[4:], p)})

        th = [threading.Thread(target=worker, args=(t,)) for t in (0, 1)]
        for t in th:
            t.start()
        for t in th:
            t.join()
        assert [results[i] for i in range(12)] == want
        pk.free()
        b2.free()
    finally:
        pool.close()


def test_real_statements(ctx, srs_2_16, srs_2_16_g2):
    import renegade_b200 as rb
    from host_circuits import private_settlement as ps
    from host_circuits import statements as st
    from host_circuits import valid_balance_create as vbc
    from renegade_b200 import circuit_types as ct
    params = rb.parse_ptau_file(ctx, srs_2_16, count=(1 << 16) + 3)
    h, tau_h = srs_2_16_g2
    ct.set_system_srs(ctx, params.powers_of_g, h, tau_h)
    try:
        vbc_inst = [vbc.create_witness_statement(seed) for seed in (3, 4, 5)]
        set_inst = [ps.create_witness_statement(seed) for seed in (61, 62)]
        items = []
        for circuit, inst, seed in ((st.ValidBalanceCreate, vbc_inst, 1), (st.IntentAndBalancePrivateSettlementCircuit, set_inst, 2)):
            got = ct.singleprover_prove_batch_with_hint(circuit, inst, rng=random.Random(seed))
            rng = random.Random(seed)
            for (w, s), (proof, hint) in zip(inst, got):
                p1, h1 = ct.singleprover_prove_with_hint(circuit, w, s, rng=rng)
                assert bytes(proof) == bytes(p1)
                assert (hint.linking_wire_poly == h1.linking_wire_poly).all()  # hence the same link proofs
                items.append((circuit, s, proof))
        ct.batch_verify_singleprover_proofs(items)
        w, s = vbc_inst[0]
        bad_w = vbc.create_witness_statement(9)[0]
        with pytest.raises(ct.ProverError) as err:
            ct.singleprover_prove_batch(st.ValidBalanceCreate, [(w, s), (bad_w, s)])  # witness 1 does not fit statement 0
        assert "[1]" in str(err.value)
    finally:
        ct.clear_key_cache()


def test_bad_arguments(ctx, oracle, pyoracle):
    from renegade_b200.backend import B200ProveItem
    circ, srs, bases, pk = make(ctx, oracle, pyoracle, 5, 2, seed=3)
    lib = ctx._lib
    st = (C.c_int * 2)()
    assert lib.b200_plonk_prove_batch(ctx._h, pk._h, None, 0, st) == 0
    assert lib.b200_plonk_prove_batch(ctx._h, pk._h, None, 2, st) == -1
    items = (B200ProveItem * 1)()
    w = np.ascontiguousarray(circ.wires)
    bl = synth.splitmix_blinders(1)
    from renegade_b200.backend import B200Proof
    proof = B200Proof()
    items[0] = B200ProveItem(w.ctypes.data, None, bl.ctypes.data, C.cast(C.pointer(proof), C.c_void_p), None, None)
    assert lib.b200_plonk_prove_batch(ctx._h, pk._h, items, 1, st) == -1  # the key takes 2 public inputs
    assert PlonkKzgSnark.prove_batch(ctx, pk, [], [], []) == ([], None, [])
    pk.free()
    bases.free()
