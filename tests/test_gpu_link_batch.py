"""Batch link proving (`b200_plonk_link_batch`, `link_proofs_batch`, `ProverPool.submit_link_batch`): k link proofs made by
one call must give, item by item, the bytes `b200_plonk_link` gives for the same inputs — proof and eta — whatever the mix
of transform sizes and layouts, the order, the chunking, the pointer kinds and the refused items around them, and without
disturbing the single link prover's or the single prover's graphs.  The inputs are built from the algebra
(`link_layouts.py`) and, for the real private match, from the restated statements."""
import ctypes as C
import random
import threading

import numpy as np
import pytest

import link_layouts as ll
from renegade_b200 import synth
from renegade_b200.backend import (B200LinkItem, GroupLayout, LinkingHint, PlonkKzgSnark, ProverPool, _link_items,
                                   link_proofs, link_proofs_batch, verify_link_proof)

pytestmark = pytest.mark.gpu

TAU = 0x1D2C3B4A59687706F5E4D3C2B1A09F8E7D6C5B4A39281706F5E4D3C2B1A0987  # conftest's SRS_2_16_TAU: srs_2_16_g2 is its G2 pair
UNSAT, INVALID = -7, -1
WRAPS = ll.BY_NAME["wraps"]


@pytest.fixture(scope="module")
def env(ctx, oracle, srs_2_16_g2):
    class E:
        pass
    e = E()
    e.ctx, e.oracle = ctx, oracle
    e.tau = oracle.int_to_limbs(TAU % ll.R * ll.MONT % ll.R)
    e.srs = oracle.srs_from_tau(e.tau, (1 << 17) + 3)
    e.bases = ctx.load_bases(e.srs)
    e.h, e.tau_h = srs_2_16_g2
    yield e
    e.bases.free()


def hint(e, vals):
    m = ll.to_mont(vals)
    xy, inf = e.ctx.msm(e.bases, m, montgomery=True)
    return LinkingHint(m, np.zeros(8, dtype=np.uint64) if inf else xy)


def layout(c):
    return GroupLayout(c.alignment, c.offset, c.size)


def triple(e, c, seed):
    a1, a2 = ll.pair(e.oracle, c, seed)
    return hint(e, a1), hint(e, a2), layout(c)


def single(e, t):
    lp, eta = link_proofs(e.ctx, e.bases, *t)
    return bytes(lp), eta.tobytes()


def batch(e, triples, ctx=None):
    proofs, etas, st = link_proofs_batch(ctx or e.ctx, e.bases, triples)
    return [(bytes(p), eta.tobytes() if eta is not None else None) for p, eta in zip(proofs, etas)], st


SENTINEL = np.uint64(0xA5A5A5A5A5A5A5A5)


def raw_batch(e, triples, edit=None):
    """the C call on items whose eta buffers and statuses hold a sentinel: (rc, statuses, proofs, etas, last error)"""
    items, keep = _link_items(e.bases, triples)
    for x in keep:
        x[5][:] = SENTINEL
    if edit:
        edit(items, keep)
    st = (C.c_int * max(1, len(keep)))(*([0x5A5A] * max(1, len(keep))))
    rc = e.ctx._lib.b200_plonk_link_batch(e.ctx._h, e.bases._h, items, len(keep), st)
    err = e.ctx._lib.b200_last_error()
    return rc, list(st)[:len(keep)], [bytes(x[4]) for x in keep], [x[5].copy() for x in keep], err


def test_every_layout_in_one_batch(env):
    """mixed N (2^4 .. 2^18), size 1, q_len 1, the whole subgroup, wrapping roots, an alignment above log2 N, len = N,
    both length orders, equal polynomials and the largest SRS: one call, the single call's and the oracle's bytes"""
    e = env
    triples = [triple(e, c, seed=0x11 + i) for i, c in enumerate(ll.CASES)]
    want = [single(e, t) for t in triples]
    got, st = batch(e, triples)
    assert st == [0] * len(ll.CASES)
    assert got == want
    for c, t, (lp, eta) in zip(ll.CASES, triples, got):
        h1, h2, _ = t
        rc, olp, oeta = e.oracle.plonk_link(h1.linking_wire_poly, h2.linking_wire_poly, h1.linking_wire_comm,
                                            h2.linking_wire_comm, c.alignment, c.offset, c.size, e.srs)
        assert rc == 0 and lp == bytes(olp) and eta == oeta.tobytes(), c.name
        assert (not any(lp)) == c.identical, c.name  # equal polynomials: identity commitments, 64 zero bytes each
    proofs, _, _ = link_proofs_batch(e.ctx, e.bases, triples)
    links = [(t[0].linking_wire_comm, t[1].linking_wire_comm, p, t[2]) for t, p in zip(triples, proofs)]
    ok, verdicts = PlonkKzgSnark.batch_verify(e.ctx, [], [], [], links, g2=(e.h, e.tau_h))
    assert ok and verdicts == [True] * len(links)
    order = list(range(len(triples)))
    random.Random(3).shuffle(order)
    got, st = batch(e, [triples[i] for i in order])
    assert st == [0] * len(order) and got == [want[i] for i in order]


def test_k_items_of_one_layout_and_a_permutation(env):
    e = env
    triples = [triple(e, WRAPS, seed=0x900 + i) for i in range(64)]
    want = [single(e, t) for t in triples]
    assert len(set(want)) == 64
    for k in (1, 2, 3, 64):
        got, st = batch(e, triples[:k])
        assert st == [0] * k and got == want[:k], k
    order = list(range(64))
    random.Random(9).shuffle(order)
    got, st = batch(e, [triples[i] for i in order])
    assert got == [want[i] for i in order]
    assert link_proofs_batch(e.ctx, e.bases, []) == ([], [], [])


def test_chunking_does_not_change_the_bytes(env, monkeypatch):
    e = env
    cases = [c for c in ll.CASES if c.name != "largest_srs"]
    triples = [triple(e, c, seed=0x300 + i) for i, c in enumerate(cases)]
    a1, a2 = ll.pair(e.oracle, WRAPS, seed=0x3FF)
    triples.insert(4, (hint(e, ll.mismatch(e.oracle, WRAPS, a1, 2, 77)), hint(e, a2), layout(WRAPS)))
    one, st1 = batch(e, triples)
    assert st1 == [UNSAT if i == 4 else 0 for i in range(len(triples))]
    for chunk in ("1", "2", "3"):
        monkeypatch.setenv("B200_LINK_BATCH_CHUNK", chunk)
        got, st = batch(e, triples)
        assert st == st1 and got == one, chunk
    monkeypatch.delenv("B200_LINK_BATCH_CHUNK")


@pytest.mark.parametrize("bad_at", [[0], [2], [4], [0, 1, 2, 3, 4]])
def test_refused_items(env, bad_at):
    """a1 + c Z_D / (X - root_j) differs from a2 on root j only: that item is refused, the others are proved"""
    e = env
    pairs = [ll.pair(e.oracle, WRAPS, seed=0x500 + i) for i in range(5)]
    honest = [(hint(e, a1), hint(e, a2), layout(WRAPS)) for a1, a2 in pairs]
    want = [single(e, t) for t in honest]
    triples = [(hint(e, ll.mismatch(e.oracle, WRAPS, pairs[i][0], i % WRAPS.size, 0xBAD + i)), honest[i][1], honest[i][2])
               if i in bad_at else honest[i] for i in range(5)]
    rc, st, proofs, etas, err = raw_batch(e, triples)
    assert rc == UNSAT and b"see statuses" in err
    assert st == [UNSAT if i in bad_at else 0 for i in range(5)]
    for i in range(5):
        if i in bad_at:
            assert proofs[i] == bytes(128) and (etas[i] == SENTINEL).all(), i
        else:
            assert (proofs[i], etas[i].tobytes()) == want[i], i
    got, _ = batch(e, triples)
    assert [g for i, g in enumerate(got) if i not in bad_at] == [w for i, w in enumerate(want) if i not in bad_at]
    assert single(e, honest[0]) == want[0]  # the context keeps proving


def test_host_pinned_and_device_pointers(env):
    import torch
    e = env
    triples = [triple(e, c, seed=0x700 + i) for i, c in enumerate(ll.CASES[:6])]
    want = [single(e, t) for t in triples]
    held = []

    def moved(h, kind):
        t = torch.from_numpy(h.linking_wire_poly.view(np.int64))
        t = t.cuda() if kind == "device" else t.pin_memory()
        held.append(t)
        return LinkingHint((t.data_ptr(), h.linking_wire_poly.shape[0]), h.linking_wire_comm)

    kinds = [("device", "host"), ("pinned", "device"), ("host", "pinned"), ("device", "device"), ("pinned", "pinned"),
             ("host", "host")]
    mixed = [(moved(a, ka) if ka != "host" else a, moved(b, kb) if kb != "host" else b, lay)
             for (a, b, lay), (ka, kb) in zip(triples, kinds)]
    torch.cuda.synchronize()
    got, st = batch(e, mixed)
    assert st == [0] * 6 and got == want


def test_single_link_proofs_and_proofs_keep_their_graphs(env, oracle, pyoracle):
    e = env
    ctx = e.ctx
    ctx.use_graphs(True)
    c = ll.Case("graphs", 6, 17, 9, 52, 47, N=64, q_len=43)
    t = triple(e, c, seed=0x6A)
    single(e, t)  # eager
    single(e, t)  # captured
    g0 = ctx.graph_launches()
    before = single(e, t)
    assert ctx.graph_launches() - g0 == 2
    circ = synth.synth_circuit(8, num_inputs=2, seed=0x6B, check=True)
    srs8 = oracle.srs_from_tau(e.tau, (1 << 8) + 3)
    b8 = ctx.load_bases(srs8)
    pk = PlonkKzgSnark.preprocess(ctx, b8, 8, circ.num_inputs, circ.selectors, circ.perm, circ.k)
    bl = synth.splitmix_blinders(0x6C)
    for _ in range(2):  # eager, captured
        PlonkKzgSnark.prove_with_link_hint(ctx, pk, circ.wires, circ.pub_inputs, bl)
    g0 = ctx.graph_launches()
    proof0, _ = PlonkKzgSnark.prove_with_link_hint(ctx, pk, circ.wires, circ.pub_inputs, bl)
    assert ctx.graph_launches() - g0 == 7
    g1 = ctx.graph_launches()
    got, st = batch(e, [t, triple(e, ll.BY_NAME["len1_far_above_len2"], seed=0x6D), t])
    assert st == [0, 0, 0] and got[0] == got[2] == before
    assert ctx.graph_launches() == g1  # a batch runs eagerly
    g2 = ctx.graph_launches()
    assert single(e, t) == before
    assert ctx.graph_launches() - g2 == 2
    g3 = ctx.graph_launches()
    proof1, _ = PlonkKzgSnark.prove_with_link_hint(ctx, pk, circ.wires, circ.pub_inputs, bl)
    assert ctx.graph_launches() - g3 == 7 and bytes(proof1) == bytes(proof0)
    pk.free()
    b8.free()


def test_pool_batches_from_two_threads(env, oracle):
    e = env
    triples = [triple(e, c, seed=0x800 + i) for i, c in enumerate(ll.CASES[:8])]
    want = [single(e, t) for t in triples]
    lay = GroupLayout(alignment=7, offset=20, size=9)
    vals = [(i * 0xD1B54A32D192ED03 + 99) % ll.R for i in range(lay.size)]
    circs = [synth.synth_circuit(lg, num_inputs=3, seed=0x80 + lg, check=True, link=(lay.alignment, lay.offset, vals))
             for lg in (8, 9)]
    bl = [synth.splitmix_blinders(0x81 + i) for i in range(2)]
    pool = ProverPool(device=0, workers=2)
    try:
        pc = pool.context(0)
        bases = pc.load_bases(e.srs)
        pks = [PlonkKzgSnark.preprocess(pc, bases, lg, c.num_inputs, c.selectors, c.perm, c.k) for lg, c in zip((8, 9), circs)]
        wires = [np.ascontiguousarray(c.wires, dtype=np.uint64) for c in circs]
        results, bundle = {}, {}

        def worker(t):
            idx = list(range(4 * t, 4 * t + 4))
            ts = pool.submit_link(bases, *triples[idx[0]])
            tb = pool.submit_link_batch(bases, [triples[i] for i in idx[1:3]])
            if t == 0:
                tu = pool.submit_bundle(bases, [(pks[i], wires[i].ctypes.data, circs[i].pub_inputs, bl[i]) for i in range(2)],
                                        [(0, 1, lay)])
            tb2 = pool.submit_link_batch(bases, [triples[idx[3]]])
            results[idx[0]] = (bytes(pool.wait(ts)), None)
            p, etas, st = pool.wait(tb)
            assert st == [0, 0]
            results.update({i: (bytes(x), y.tobytes()) for i, x, y in zip(idx[1:3], p, etas)})
            if t == 0:
                bundle["out"] = pool.wait(tu)
            p, etas, st = pool.wait(tb2)
            assert st == [0]
            results[idx[3]] = (bytes(p[0]), etas[0].tobytes())

        th = [threading.Thread(target=worker, args=(t,)) for t in (0, 1)]
        for t in th:
            t.start()
        for t in th:
            t.join()
        assert sorted(results) == list(range(8))
        for i in range(8):
            assert results[i][0] == want[i][0] and results[i][1] in (None, want[i][1]), i
        proofs, polys, links = bundle["out"]
        hints = [LinkingHint(polys[i], np.array(proofs[i].wires_poly_comms[0], dtype=np.uint64)) for i in range(2)]
        assert bytes(links[0]) == single(e, (hints[0], hints[1], lay))[0]
        for pk in pks:
            pk.free()
        bases.free()
    finally:
        pool.close()


def test_real_private_match(ctx, srs_2_16, srs_2_16_g2):
    """the four link proofs of one private match (two INTENT AND BALANCE VALIDITY and two OUTPUT BALANCE VALIDITY hints
    against the PRIVATE SETTLEMENT hint, N = 2^15 and 2^14) as one batch: the four single link proofs, byte for byte,
    each accepted by the pairing against the SRS's [tau]_2"""
    import renegade_b200 as rb
    from host_circuits import intent_and_balance_validity as val
    from host_circuits import output_balance_validity as obv
    from host_circuits import private_settlement as ps
    from host_circuits import statements as st
    from renegade_b200 import circuit_types as ct
    real_srs = rb.parse_ptau_file(ctx, srs_2_16, count=(1 << 16) + 3).powers_of_g
    h, tau_h = srs_2_16_g2
    ct.set_system_srs(ctx, real_srs, h, tau_h)
    try:
        parties, _ = ps.create_witness_statement(seed=61)
        validity = [val.create_witness_statement(seed=70 + i, intent=parties[i].intent, balance=parties[i].input_balance)
                    for i in (0, 1)]
        out_validity = [obv.create_witness_statement(80 + i, parties[i].output_balance) for i in (0, 1)]
        parties, statement = ps.create_witness_statement(
            seed=61, linked=[(validity[i][0].new_amount_public_share, validity[i][0].post_match_balance_shares,
                              out_validity[i][0].post_match_balance_shares) for i in (0, 1)])
        S = st.IntentAndBalancePrivateSettlementCircuit
        _, sh = ct.singleprover_prove_with_hint(S, parties, statement)
        layouts = S.get_circuit_layout()
        triples = []
        for i in (0, 1):
            for Circ, (w, s_), gid in ((st.IntentAndBalanceValidityCircuit, validity[i], ps.PARTY_LINKS[i]),
                                       (st.OutputBalanceValidityCircuit, out_validity[i], ps.OUTPUT_LINKS[i])):
                _, hnt = ct.singleprover_prove_with_hint(Circ, w, s_)
                triples.append((hnt, sh, GroupLayout(layouts[gid].alignment, layouts[gid].offset, layouts[gid].size)))
        assert len({t[0].linking_wire_poly.shape[0] for t in triples} | {sh.linking_wire_poly.shape[0]}) > 1  # mixed N
        want = [link_proofs(ctx, real_srs, *t) for t in triples]
        proofs, etas, sts = link_proofs_batch(ctx, real_srs, triples)
        assert sts == [0] * 4
        for (lp, eta), p, et, (a, b, lay) in zip(want, proofs, etas, triples):
            assert bytes(p) == bytes(lp) and et.tobytes() == eta.tobytes()
            assert verify_link_proof(a.linking_wire_comm, b.linking_wire_comm, p, lay, h, tau_h)
    finally:
        ct.clear_key_cache()


@pytest.mark.parametrize("bad", ["size_zero", "size_is_len", "size_above_group", "alignment", "longer_than_srs", "null_a1",
                                 "null_a2", "null_comm1", "null_comm2", "null_proof"])
def test_argument_errors_fail_the_call_before_any_work(env, bad):
    e = env
    triples = [triple(e, WRAPS, seed=0x400 + i) for i in range(3)]
    long_poly = np.zeros((e.srs.shape[0] + 1, 4), dtype=np.uint64)

    def edit(items, keep):
        it = items[1]
        if bad == "size_zero":
            it.size = 0
        elif bad == "size_is_len":
            it.size = max(it.len1, it.len2)
        elif bad == "size_above_group":  # 2^3 + 1 roots at alignment 3, below the length 20
            it.size = (1 << it.alignment) + 1
        elif bad == "alignment":
            it.alignment = 29
        elif bad == "longer_than_srs":
            it.a1, it.len1 = long_poly.ctypes.data, long_poly.shape[0]
        else:
            setattr(it, bad[5:], None)
    rc, st, proofs, etas, err = raw_batch(e, triples, edit)
    assert rc == INVALID and b"item 1" in err, bad
    assert st == [0x5A5A] * 3 and proofs == [bytes(128)] * 3 and all((x == SENTINEL).all() for x in etas)
    lib = e.ctx._lib
    assert lib.b200_plonk_link_batch(e.ctx._h, e.bases._h, None, 2, None) == INVALID
    assert lib.b200_plonk_link_batch(e.ctx._h, None, (B200LinkItem * 1)(), 1, None) == INVALID
    assert lib.b200_plonk_link_batch(e.ctx._h, e.bases._h, None, 0, None) == 0
