"""Settlement jobs (`b200_plonk_prove_settlement[_witness]`, `b200_pool_submit_settlement[_witness]`,
`b200_box_submit_settlement[_witness]`): a settlement statement proved and linked, in one call, against hints kept from
validity proofs made in earlier calls.  Every proof, link proof and eta equals the single calls (`b200_plonk_prove[_witness]`
+ `b200_plonk_link`); a stale hint fails only its own link; an unsatisfied settlement fails everything and leaves the
context and the pool usable; argument errors launch nothing and queue nothing."""
import ctypes as C
import threading

import numpy as np
import pytest

from renegade_b200 import _lib, synth
from renegade_b200.backend import (GroupLayout, LinkingHint, PlonkKzgSnark, ProverBox, ProverError, ProverPool,
                                   SettlementLink, VerifyingKey, link_proofs, link_proofs_batch)
from test_gpu_prove_witness import TAU, unsatisfying
from test_gpu_witness_jobs import Setup, private_match
from test_prove_witness_cpu import wiring_permutation

pytestmark = pytest.mark.gpu
OK, INVALID, UNSAT = _lib.B200_OK, _lib.B200_ERR_INVALID, _lib.B200_ERR_UNSATISFIED


def intent_only():
    """INTENT ONLY PUBLIC SETTLEMENT (2^9) and the INTENT ONLY VALIDITY proof (2^13) of the same intent; link: 1 -> 0."""
    from host_circuits import intent_only as io
    intent = io.create_public_settlement_witness_statement(51)[0].intent
    settlement = io.IntentOnlyPublicSettlementCircuit.build(*io.create_public_settlement_witness_statement(54, intent))
    lay = settlement.get_circuit_layout()[io.INTENT_ONLY_SETTLEMENT_LINK]
    validity = io.IntentOnlyValidityCircuit.build(*io.create_validity_witness_statement(52, intent), lay)
    other = io.IntentOnlyValidityCircuit.build(*io.create_validity_witness_statement(57), lay)  # another order's
    circs = [c.finalize_for_arithmetization() for c in (settlement, validity, other)]
    return circs, [(1, 0, GroupLayout(lay.alignment, lay.offset, lay.size))]


def private():
    """PRIVATE SETTLEMENT (2^12) against the four validity hints (2^14 + 2, 2^13 + 2) of its two parties."""
    return private_match()


class Shape:
    """A settlement (proof 0), its hint proofs made in earlier calls, and the single calls' results to compare with."""

    def __init__(self, ctx, oracle, pyoracle, circs, links):
        self.s = Setup(ctx, oracle, pyoracle, circs, links)
        self.ctx, self.circs = ctx, circs
        self.bl = [synth_blinders(9000 + i) for i in range(len(circs))]
        self.hints = {}
        for j in {a for a, _, _ in links} | set(range(1, len(circs))):
            _, hint, _ = PlonkKzgSnark.prove_witness(ctx, self.s.pks[j], circs[j].witness, self.bl[j])
            self.hints[j] = hint
        self.links = [(self.hints[a], lay) for a, _, lay in links]
        self.ref = self.single_calls(self.bl[0], self.links)

    def single_calls(self, bl, links):
        """(proof, settlement hint, [(link proof, eta)]) of b200_plonk_prove + b200_plonk_link"""
        c = self.circs[0]
        proof, hint = PlonkKzgSnark.prove_with_link_hint(self.ctx, self.s.pks[0], self.s.tables[0], c.pub_inputs, bl)
        return proof, hint, [link_proofs(self.ctx, self.s.bases, h, hint, lay) for h, lay in links]

    def check(self, proof, lps, statuses, ref=None):
        ref = ref or self.ref
        assert statuses == [OK] * (len(lps) + 1)
        assert bytes(proof) == bytes(ref[0])
        assert [bytes(x) for x in lps] == [bytes(x) for x, _ in ref[2]]

    def free(self):
        self.s.free()


def synth_blinders(seed):
    return synth.splitmix_blinders(seed)


@pytest.fixture(scope="module", params=["private", "intent_only"])
def shape(request, ctx, oracle, pyoracle):
    s = Shape(ctx, oracle, pyoracle, *(private() if request.param == "private" else intent_only()))
    yield s
    s.free()


@pytest.fixture(scope="module")
def io_shape(ctx, oracle, pyoracle):
    s = Shape(ctx, oracle, pyoracle, *intent_only())
    yield s
    s.free()


@pytest.fixture(scope="module")
def pool():
    p = ProverPool(0, workers=4)
    yield p
    p.close()


def raw(ctx, shape, links, witness=False, wires=None, bl=None, n_links=None, srs=None, pk=None):
    """The C entry point with every output: (rc, proof, link_poly, [link proofs], [etas], statuses)"""
    s, c = shape.s, shape.circs[0]
    bl = shape.bl[0] if bl is None else bl
    arr = (SettlementLink * max(1, len(links)))()
    held, lps, etas = [], [], []
    for i, (hint, lay) in enumerate(links):
        poly = np.ascontiguousarray(hint.linking_wire_poly, dtype=np.uint64)
        comm = np.ascontiguousarray(hint.linking_wire_comm, dtype=np.uint64)
        lp, eta = _lib.STRUCTS["b200_link_proof"](), np.full(4, 0xEE, dtype=np.uint64)
        arr[i] = SettlementLink(poly.ctypes.data_as(C.c_void_p), poly.shape[0], comm.ctypes.data_as(C.c_void_p), lay.alignment,
                                lay.offset, lay.size, C.cast(C.pointer(lp), C.c_void_p), eta.ctypes.data_as(C.c_void_p))
        held += [poly, comm]
        lps.append(lp)
        etas.append(eta)
    proof = _lib.STRUCTS["b200_proof"]()
    link_poly = np.zeros((c.n + 2, 4), dtype=np.uint64)
    st = (C.c_int * (len(links) + 1))(*([99] * (len(links) + 1)))
    lib, p = ctx._lib, lambda a: a.ctypes.data_as(C.c_void_p)  # noqa: E731
    srs = s.bases._h if srs is None else srs
    pk = s.pks[0]._h if pk is None else pk
    n = len(links) if n_links is None else n_links
    if witness:
        pub = np.zeros((c.num_inputs, 4), dtype=np.uint64)
        rc = lib.b200_plonk_prove_settlement_witness(ctx._h, srs, pk, p(np.ascontiguousarray(c.witness)) if wires is None else wires,
                                                     p(bl), C.byref(proof), p(link_poly), p(pub), arr, n, st)
    else:
        pi = np.ascontiguousarray(c.pub_inputs, dtype=np.uint64)
        rc = lib.b200_plonk_prove_settlement(ctx._h, srs, pk, p(s.tables[0]) if wires is None else wires, p(pi), p(bl),
                                             C.byref(proof), p(link_poly), arr, n, st)
    return rc, proof, link_poly, lps, etas, list(st)


def test_every_entry_point_equals_single_calls(ctx, pool, shape, srs_2_16_g2):
    s, c, ref = shape.s, shape.circs[0], shape.ref
    pk, bases = s.pks[0], s.bases
    # context: bytes of the proof, the settlement hint, every link proof and eta
    for witness in (False, True):
        rc, proof, link_poly, lps, etas, st = raw(ctx, shape, shape.links, witness=witness)
        assert rc == OK and st == [OK] * (len(lps) + 1)
        assert bytes(proof) == bytes(ref[0]) and link_poly.tobytes() == ref[1].linking_wire_poly.tobytes()
        for lp, eta, (rlp, reta) in zip(lps, etas, ref[2]):
            assert bytes(lp) == bytes(rlp) and eta.tobytes() == reta.tobytes()
    res = [PlonkKzgSnark.prove_settlement(ctx, bases, pk, s.tables[0], c.pub_inputs, shape.bl[0], shape.links),
           PlonkKzgSnark.prove_settlement_witness(ctx, bases, pk, c.witness, shape.bl[0], shape.links),
           pool.wait(pool.submit_settlement(bases, pk, s.tables[0], c.pub_inputs, shape.bl[0], shape.links)),
           pool.wait(pool.submit_settlement_witness(bases, pk, c.witness, shape.bl[0], shape.links))]
    for r in res:
        shape.check(*r[:3])
    for r in res[1::2]:
        assert r[3].tobytes() == np.ascontiguousarray(c.pub_inputs).tobytes()
    # one batch verification accepts the proof and every link proof
    vk = VerifyingKey.from_proving_key(pk, *srs_2_16_g2)
    s_comm = np.array(ref[0].wires_poly_comms[0], dtype=np.uint64)
    lps = res[2][1]
    ok, verdicts = PlonkKzgSnark.batch_verify(ctx, [vk], [c.pub_inputs], [res[2][0]],
                                              [(h.linking_wire_comm, s_comm, lp, lay) for (h, lay), lp in zip(shape.links, lps)])
    assert ok and all(verdicts)


def test_intent_only_equals_the_oracle(io_shape, oracle, pyoracle):
    shape = io_shape
    c, hint = shape.circs[0], shape.links[0][0]
    srs = oracle.srs_from_tau(oracle.int_to_limbs(pyoracle.to_mont(TAU % pyoracle.R, pyoracle.R)), shape.s.bases.__len__())
    opk = oracle.plonk_preprocess(c.log_n, c.selectors, wiring_permutation(c.wire_vars), c.k, srs)
    rc, oproof, _, olink = oracle.plonk_prove(c.log_n, c.num_inputs, c.k, opk, shape.s.tables[0], c.pub_inputs, shape.bl[0],
                                              srs, want_link_poly=True)
    proof, lps, st = PlonkKzgSnark.prove_settlement(shape.ctx, shape.s.bases, shape.s.pks[0], shape.s.tables[0],
                                                    c.pub_inputs, shape.bl[0], shape.links)
    assert rc == 0 and st == [OK, OK] and bytes(proof) == bytes(oproof)
    lay = shape.links[0][1]
    s_comm = np.array(proof.wires_poly_comms[0], dtype=np.uint64)
    rc, olp, _ = oracle.plonk_link(hint.linking_wire_poly, olink, hint.linking_wire_comm, s_comm, lay.alignment, lay.offset,
                                   lay.size, srs)
    assert rc == 0 and bytes(lps[0]) == bytes(olp)
    tau = oracle.int_to_limbs(pyoracle.to_mont(TAU % pyoracle.R, pyoracle.R))
    assert oracle.plonk_link_verify_known_tau(hint.linking_wire_comm, s_comm, lay.alignment, lay.offset, lay.size,
                                              oracle.LinkProof.from_buffer_copy(bytes(lps[0])), tau)


def test_stale_hints(ctx, pool, oracle, pyoracle, srs_2_16_g2):
    shape = Shape(ctx, oracle, pyoracle, *private())
    try:
        stale = shape.links[1][0]  # party 1's validity hint: another order's
        for pos in (0, 2, 3):      # first, middle, last
            links = list(shape.links)
            links[pos] = (stale, links[pos][1])
            for r in (PlonkKzgSnark.prove_settlement_witness(ctx, shape.s.bases, shape.s.pks[0], shape.circs[0].witness,
                                                             shape.bl[0], links),
                      pool.wait(pool.submit_settlement(shape.s.bases, shape.s.pks[0], shape.s.tables[0],
                                                       shape.circs[0].pub_inputs, shape.bl[0], links))):
                proof, lps, st = r[:3]
                assert st == [OK if i != pos + 1 else UNSAT for i in range(5)]
                assert bytes(proof) == bytes(shape.ref[0]) and bytes(lps[pos]) == bytes(64 * 2)
                assert all(bytes(lps[i]) == bytes(shape.ref[2][i][0]) for i in range(4) if i != pos)
            rc, *_ = raw(ctx, shape, links)
            assert rc == UNSAT and f"link(s) {pos} " in _lib.load().b200_last_error().decode()
        # the right polynomial with a wrong commitment: exactly b200_plonk_link's output, which the verifier rejects
        h0, lay0 = shape.links[0]
        wrong = LinkingHint(h0.linking_wire_poly, shape.links[1][0].linking_wire_comm)
        _, lps, st = PlonkKzgSnark.prove_settlement(ctx, shape.s.bases, shape.s.pks[0], shape.s.tables[0],
                                                    shape.circs[0].pub_inputs, shape.bl[0], [(wrong, lay0)])
        direct, _ = link_proofs(ctx, shape.s.bases, wrong, shape.ref[1], lay0)
        assert st == [OK, OK] and bytes(lps[0]) == bytes(direct)
        s_comm = np.array(shape.ref[0].wires_poly_comms[0], dtype=np.uint64)
        ok, verdicts = PlonkKzgSnark.batch_verify(ctx, [], [], [], [(wrong.linking_wire_comm, s_comm, lps[0], lay0)],
                                                  g2=srs_2_16_g2)
        assert not ok and verdicts == [False]
    finally:
        shape.free()


def test_unsatisfied_settlement(ctx, pool, io_shape):
    shape = io_shape
    c = shape.circs[0]
    bad = np.ascontiguousarray(unsatisfying(c))
    rc, proof, _, lps, etas, st = raw(ctx, shape, shape.links, witness=True, wires=bad.ctypes.data_as(C.c_void_p))
    assert rc == UNSAT and st == [UNSAT, UNSAT]
    assert bytes(proof) == bytes(len(bytes(proof))) and bytes(lps[0]) == bytes(128)
    assert etas[0].tobytes() == np.full(4, 0xEE, dtype=np.uint64).tobytes()  # not written
    assert "does not satisfy" in _lib.load().b200_last_error().decode()
    proof, lps, st, _ = pool.wait(pool.submit_settlement_witness(shape.s.bases, shape.s.pks[0], bad, shape.bl[0], shape.links))
    assert st == [UNSAT, UNSAT] and bytes(proof) == bytes(len(bytes(proof))) and bytes(lps[0]) == bytes(128)
    # the context and the pool go on with correct bytes
    shape.check(*PlonkKzgSnark.prove_settlement_witness(ctx, shape.s.bases, shape.s.pks[0], c.witness, shape.bl[0],
                                                        shape.links)[:3])
    shape.check(*pool.wait(pool.submit_settlement_witness(shape.s.bases, shape.s.pks[0], c.witness, shape.bl[0],
                                                          shape.links))[:3])


def test_argument_errors(ctx, pool, io_shape):
    shape = io_shape
    s, c = shape.s, shape.circs[0]
    h, lay = shape.links[0]
    lib = _lib.load()
    table_pk = PlonkKzgSnark.preprocess(ctx, s.bases, c.log_n, c.num_inputs, c.selectors, wiring_permutation(c.wire_vars), c.k)
    long_hint = LinkingHint(np.zeros((len(s.bases) + 1, 4), dtype=np.uint64), h.linking_wire_comm)
    cases = [([(h, GroupLayout(lay.alignment, lay.offset, 0))], {}, b"link 0: bad group layout"),
             ([(h, GroupLayout(lay.alignment, lay.offset, h.linking_wire_poly.shape[0]))], {}, b"link 0: bad group layout"),
             ([(h, lay), (h, GroupLayout(29, lay.offset, lay.size))], {}, b"link 1: bad group layout"),
             ([(h, lay), (long_hint, lay)], {}, b"link 1: bad group layout"),
             ([(h, lay)], {"srs": C.c_void_p(0)}, None),
             ([(h, lay)], {"pk": table_pk._h, "witness": True}, b"no wiring")]
    k0, st0 = ctx.kernel_launches(), pool.stats()
    for links, kw, msg in cases:
        rc, proof, link_poly, lps, etas, st = raw(ctx, shape, links, **kw)
        assert rc == INVALID, (links, kw)
        if msg:
            assert msg in lib.b200_last_error(), (msg, lib.b200_last_error())
        assert bytes(proof) == bytes(len(bytes(proof))) and not link_poly.any() and st == [99] * len(st)
        assert all(bytes(x) == bytes(128) for x in lps) and all((e == 0xEE).all() for e in etas)
    # NULL pointers inside a link, and a NULL links array with n_links > 0
    for field in ("hint_poly", "hint_comm", "proof"):
        arr = (SettlementLink * 1)()
        poly, comm = np.ascontiguousarray(h.linking_wire_poly), np.ascontiguousarray(h.linking_wire_comm)
        lp = _lib.STRUCTS["b200_link_proof"]()
        arr[0] = SettlementLink(poly.ctypes.data_as(C.c_void_p), poly.shape[0], comm.ctypes.data_as(C.c_void_p), lay.alignment,
                                lay.offset, lay.size, C.cast(C.pointer(lp), C.c_void_p), None)
        setattr(arr[0], field, None)
        proof = _lib.STRUCTS["b200_proof"]()
        pi, bl = np.ascontiguousarray(c.pub_inputs, dtype=np.uint64), shape.bl[0]
        p = lambda a: a.ctypes.data_as(C.c_void_p)  # noqa: E731
        assert lib.b200_plonk_prove_settlement(ctx._h, s.bases._h, s.pks[0]._h, p(s.tables[0]), p(pi), p(bl), C.byref(proof),
                                               None, arr, 1, None) == INVALID
        assert b"link 0 has a NULL" in lib.b200_last_error()
        bp = _lib.STRUCTS["b200_bundle_proof"](s.pks[0]._h, p(s.tables[0]), p(pi), c.num_inputs, p(bl),
                                               C.cast(C.pointer(proof), C.c_void_p), None)
        t = C.c_uint64()
        assert lib.b200_pool_submit_settlement(pool._h, s.bases._h, C.byref(bp), arr, 1, None, C.byref(t)) == INVALID
        assert lib.b200_pool_submit_settlement(pool._h, s.bases._h, C.byref(bp), None, 1, None, C.byref(t)) == INVALID
        assert bytes(proof) == bytes(len(bytes(proof)))
    # the pool refuses at submit what the context refuses, and the Python checks come first
    for links in ([(h, GroupLayout(29, lay.offset, lay.size))], [(long_hint, lay)]):
        with pytest.raises(ProverError):
            pool.submit_settlement(s.bases, s.pks[0], s.tables[0], c.pub_inputs, shape.bl[0], links)
    with pytest.raises(ProverError, match="no wiring"):
        pool.submit_settlement_witness(s.bases, table_pk, c.witness, shape.bl[0], shape.links)
    assert ctx.kernel_launches() == k0 and pool.stats() == st0 and st0["queued"] == 0
    table_pk.free()


def test_pointer_kinds_and_link_counts(ctx, pool, io_shape):
    """numpy, pinned, device and device + 16 bytes hints and witnesses mixed in one job; 0, 1 and 65 links."""
    import torch
    shape = io_shape
    s, c = shape.s, shape.circs[0]
    h, lay = shape.links[0]
    poly = np.ascontiguousarray(h.linking_wire_poly)
    pinned = torch.from_numpy(poly.view(np.int64)).pin_memory()
    dev = torch.from_numpy(poly.view(np.int64)).cuda()
    dev16 = torch.zeros(poly.size + 2, dtype=torch.int64, device="cuda")
    dev16[2:] = torch.from_numpy(poly.view(np.int64).reshape(-1)).cuda()
    wit = np.ascontiguousarray(c.witness)
    wdev = torch.from_numpy(wit.view(np.int64)).cuda()
    torch.cuda.synchronize()
    kinds = [poly, (pinned.data_ptr(), poly.shape[0]), (dev.data_ptr(), poly.shape[0]), (dev16.data_ptr() + 16, poly.shape[0])]
    links = [(LinkingHint(k, h.linking_wire_comm), lay) for k in kinds]
    ref = shape.single_calls(shape.bl[0], [(h, lay)])
    for witness in (wit, wdev.data_ptr()):
        for r in (PlonkKzgSnark.prove_settlement_witness(ctx, s.bases, s.pks[0], witness, shape.bl[0], links),
                  pool.wait(pool.submit_settlement_witness(s.bases, s.pks[0], witness, shape.bl[0], links, keep=(dev, dev16)))):
            proof, lps, st = r[:3]
            assert st == [OK] * 5 and bytes(proof) == bytes(ref[0])
            assert all(bytes(x) == bytes(ref[2][0][0]) for x in lps)
    for n in (0, 1, 65):
        proof, lps, st = PlonkKzgSnark.prove_settlement(ctx, s.bases, s.pks[0], s.tables[0], c.pub_inputs, shape.bl[0],
                                                        [(h, lay)] * n)
        assert st == [OK] * (n + 1) and bytes(proof) == bytes(ref[0]) and len(lps) == n
        assert all(bytes(x) == bytes(ref[2][0][0]) for x in lps)


def test_steady_state_graphs_and_kernels(ctx, oracle, pyoracle):
    shape = Shape(ctx, oracle, pyoracle, *private())
    try:
        s, c = shape.s, shape.circs[0]
        args = (s.bases, s.pks[0], s.tables[0], c.pub_inputs, shape.bl[0], shape.links)
        for _ in range(2):
            PlonkKzgSnark.prove_settlement(ctx, *args)
        g0, k0 = ctx.graph_launches(), ctx.kernel_launches()
        shape.check(*PlonkKzgSnark.prove_settlement(ctx, *args))
        g1, k1 = ctx.graph_launches(), ctx.kernel_launches()
        assert g1 - g0 == 7
        PlonkKzgSnark.prove_with_link_hint(ctx, s.pks[0], s.tables[0], c.pub_inputs, shape.bl[0])
        link_proofs_batch(ctx, s.bases, [(hh, shape.ref[1], lay) for hh, lay in shape.links])
        assert ctx.kernel_launches() - k1 == k1 - k0
    finally:
        shape.free()


def test_two_threads_interleaved_with_other_jobs(pool, io_shape):
    shape = io_shape
    s, c = shape.s, shape.circs[0]
    h, lay = shape.links[0]
    errors = []

    def run(seed):
        try:
            for i in range(3):
                bl = synth_blinders(seed + i)
                t_set = pool.submit_settlement_witness(s.bases, s.pks[0], c.witness, bl, shape.links)
                t_one = pool.submit_prove(s.pks[1], s.tables[1].ctypes.data, shape.circs[1].pub_inputs, shape.bl[1],
                                          keep=s.tables[1])
                t_lb = pool.submit_link_batch(s.bases, [(h, shape.ref[1], lay)] * 3)
                got = pool.wait(t_set)
                one = pool.wait(t_one)
                lb = pool.wait(t_lb)
                results.append((bl.tobytes(), bytes(got[0]), [bytes(x) for x in got[1]], got[2], bytes(one),
                                [bytes(x) for x in lb[0]]))
        except Exception as e:  # reported by the main thread
            errors.append(e)

    results = []
    threads = [threading.Thread(target=run, args=(9500 + 100 * t,)) for t in range(2)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert not errors, errors
    one_ref = PlonkKzgSnark.prove_with_link_hint(shape.ctx, s.pks[1], s.tables[1], shape.circs[1].pub_inputs, shape.bl[1])[0]
    for bl_bytes, proof, lps, st, one, lb in results:
        ref = shape.single_calls(np.frombuffer(bl_bytes, dtype=np.uint64).reshape(17, 4), shape.links)
        assert st == [OK, OK] and proof == bytes(ref[0]) and lps == [bytes(x) for x, _ in ref[2]]
        assert one == bytes(one_ref) and lb == [bytes(shape.ref[2][0][0])] * 3
    assert len(results) == 6


def test_box(io_shape, oracle, pyoracle):
    import torch
    shape = io_shape
    c = shape.circs[0]
    devices = [0, 1] if torch.cuda.device_count() >= 2 else [0, 0]
    box = ProverBox(devices, workers_per_device=2)
    try:
        tau = oracle.int_to_limbs(pyoracle.to_mont(TAU % pyoracle.R, pyoracle.R))
        srs = box.load_srs(oracle.srs_from_tau(tau, len(shape.s.bases)))
        pk = box.preprocess_wiring(srs, c.log_n, c.num_inputs, c.selectors, c.wire_vars, c.num_vars, c.k)
        for r in (box.wait(box.submit_settlement(srs, pk, shape.s.tables[0], c.pub_inputs, shape.bl[0], shape.links)),
                  box.wait(box.submit_settlement_witness(srs, pk, c.witness, shape.bl[0], shape.links))):
            shape.check(*r[:3])
        h, lay = shape.links[0]
        last = len(devices) - 1
        with torch.cuda.device(devices[last]):
            dev = torch.from_numpy(np.ascontiguousarray(h.linking_wire_poly).view(np.int64)).cuda()
            torch.cuda.synchronize()
        link = [(LinkingHint((dev.data_ptr(), h.linking_wire_poly.shape[0]), h.linking_wire_comm), lay)]
        t = box.submit_settlement_witness(srs, pk, c.witness, shape.bl[0], link, keep=dev)
        assert devices[box.ticket_device(t)] == devices[last]
        shape.check(*box.wait(t)[:3])
        if devices == [0, 1]:  # device pointers on two devices cannot make one job
            with torch.cuda.device(0):
                wdev = torch.from_numpy(np.ascontiguousarray(c.witness).view(np.int64)).cuda()
                torch.cuda.synchronize()
            with pytest.raises(ProverError) as err:
                box.submit_settlement_witness(srs, pk, wdev.data_ptr(), shape.bl[0], link)
            assert err.value.code == INVALID and "two devices" in str(err.value)
        with pytest.raises(ProverError):  # a key of another box
            box.submit_settlement(srs, shape.s.pks[0]._h, shape.s.tables[0], c.pub_inputs, shape.bl[0], shape.links)
        box.free_pk(pk)
        box.free_srs(srs)
    finally:
        box.close()

