"""The express lane (include/b200express.h): jobs of every kind moved by ticket from a pool's or a box's normal queue to
its express queue, and run there on express workers whose streams outrank the normal workers'.  Every output and status
equals the bare-context call on the same inputs and blinders; `wait_info` shows where each job ran and in which order the
jobs finished, so placement and ordering are checked without timing anything.

A job under test stays queued until it is expedited because the pool's one normal worker is busy with a long blocker (a
witness batch of a 2^14 circuit) that has already started, and the express worker is idle when the job reaches it."""
import ctypes as C
import threading
import time

import numpy as np
import pytest

from renegade_b200 import _lib, synth
from renegade_b200.backend import (GroupLayout, LinkingHint, PlonkKzgSnark, ProverBox, ProverPool, VerifyingKey, link_proofs,
                                   link_proofs_batch)
from test_gpu_prove_witness import TAU, load_srs, unsatisfying
from test_gpu_witness_jobs import Setup, synthetic

pytestmark = pytest.mark.gpu
OK, INVALID = _lib.B200_OK, _lib.B200_ERR_INVALID
BLOCKER_LOG_N, BLOCKER_K = 14, 96
EXPRESS = 1  # worker index of the first express worker of a pool with one normal worker


class Env:
    """The synthetic shape (2^10, 2^11, 2^10; links 0 -> 1 and 2 -> 1) proved on the session context, and a blocker."""

    def __init__(self, ctx, oracle, pyoracle, g2):
        self.ctx, self.h, self.tau_h = ctx, g2[0], g2[1]
        self.s = Setup(ctx, oracle, pyoracle, *synthetic())
        self.bl = [synth.splitmix_blinders(7300 + j) for j in range(len(self.s.circs))]
        self.proofs, self.hints, self.pubs = [], [], []
        for pk, c, b in zip(self.s.pks, self.s.circs, self.bl):
            proof, hint, pub = PlonkKzgSnark.prove_witness(ctx, pk, c.witness, b)
            self.proofs.append(proof)
            self.hints.append(hint)
            self.pubs.append(pub)
        self.link_proofs = [link_proofs(ctx, self.s.bases, self.hints[a], self.hints[b], lay)[0] for a, b, lay in self.s.links]
        self.vks = [VerifyingKey.from_proving_key(pk, self.h, self.tau_h) for pk in self.s.pks]
        bc = synth.synth_circuit(BLOCKER_LOG_N, num_inputs=2, seed=7390)
        self.blocker_circ = bc
        self.blocker_bases = load_srs(ctx, oracle, pyoracle, bc.n)
        self.blocker_pk = PlonkKzgSnark.preprocess_wiring(ctx, self.blocker_bases, bc.log_n, bc.num_inputs, bc.selectors,
                                                          bc.wire_vars, bc.num_vars, bc.k)
        self.blocker_bl = [synth.splitmix_blinders(7400 + i) for i in range(BLOCKER_K)]

    def block(self, pool):
        """Occupy the pool's normal worker: a fresh long job that has started once this returns."""
        t = pool.submit_prove_witness_batch(self.blocker_pk, [self.blocker_circ.witness] * BLOCKER_K, self.blocker_bl)
        while pool.stats()["queued"]:
            time.sleep(0.0005)
        return t

    def free(self):
        self.blocker_pk.free()
        self.blocker_bases.free()
        self.s.free()


@pytest.fixture(scope="module")
def env(ctx, oracle, pyoracle, srs_2_16_g2):
    e = Env(ctx, oracle, pyoracle, srs_2_16_g2)
    yield e
    e.free()


def as_bytes(x):
    """A job's result as comparable bytes, whatever its nesting."""
    if x is None or isinstance(x, (int, bool, np.integer, np.bool_)):
        return x
    if isinstance(x, np.ndarray):
        return x.tobytes()
    if isinstance(x, LinkingHint):
        return (x.linking_wire_poly.tobytes(), np.asarray(x.linking_wire_comm, dtype=np.uint64).tobytes())
    if isinstance(x, (list, tuple)):
        return [as_bytes(v) for v in x]
    return bytes(x)


def kinds(e):
    """(name, submit(pool) -> ticket, bare() -> the bare context's result, jobs the ticket queues) for every job kind."""
    s, ctx, bl = e.s, e.ctx, e.bl
    c0, c1 = s.circs[0], s.circs[1]
    pk0, pk1 = s.pks[0], s.pks[1]
    bad_table = np.ascontiguousarray(unsatisfying(c1)[c1.wire_vars])
    tables1 = [s.tables[1], bad_table, s.tables[1]]
    bls3 = [synth.splitmix_blinders(7500 + i) for i in range(3)]
    a, b, lay = s.links[0]
    stale = GroupLayout(lay.alignment, lay.offset + 1, lay.size)
    triples = [(e.hints[a], e.hints[b], lay), (e.hints[a], e.hints[b], stale), (e.hints[2], e.hints[1], lay)]
    bundle_tables = [(pk, t.ctypes.data, c.pub_inputs, b_) for pk, t, c, b_ in zip(s.pks, s.tables, s.circs, bl)]
    bundle_witness = [(pk, c.witness, b_) for pk, c, b_ in zip(s.pks, s.circs, bl)]
    settle_links = [(e.hints[0], lay), (e.hints[2], s.links[1][2])]
    items = [(e.vks[j], e.pubs[j], e.proofs[j]) for j in range(3)]
    vlinks = [(e.hints[a_].linking_wire_comm, e.hints[b_].linking_wire_comm, lp, l_)
              for (a_, b_, l_), lp in zip(s.links, e.link_proofs)]
    vargs = ([i[0] for i in items], [i[1] for i in items], [i[2] for i in items], vlinks)
    g2 = (e.h, e.tau_h)

    def bundle_bare():
        proofs, polys = [], []
        for pk, t, c, b_ in zip(s.pks, s.tables, s.circs, bl):
            p, h_ = PlonkKzgSnark.prove_with_link_hint(ctx, pk, t, c.pub_inputs, b_)
            proofs.append(p)
            polys.append(h_.linking_wire_poly)
        hs = [LinkingHint(linking_wire_poly=polys[j], linking_wire_comm=np.array(proofs[j].wires_poly_comms[0], dtype=np.uint64))
              for j in range(3)]
        return proofs, polys, [link_proofs(ctx, s.bases, hs[a_], hs[b_], l_)[0] for a_, b_, l_ in s.links]

    return [
        ("prove", lambda p: p.submit_prove(pk0, s.tables[0].ctypes.data, c0.pub_inputs, bl[0], with_link_poly=True,
                                           keep=s.tables[0]),
         lambda: (lambda r: (r[0], r[1].linking_wire_poly))(PlonkKzgSnark.prove_with_link_hint(ctx, pk0, s.tables[0],
                                                                                                c0.pub_inputs, bl[0])), 1),
        ("prove_witness", lambda p: p.submit_prove_witness(pk0, c0.witness, bl[0], with_link_poly=True),
         lambda: (lambda r: (r[0], r[1].linking_wire_poly, r[2]))(PlonkKzgSnark.prove_witness(ctx, pk0, c0.witness, bl[0])), 1),
        ("prove_batch", lambda p: p.submit_prove_batch(pk1, tables1, [c1.pub_inputs] * 3, bls3, link_hints=True),
         lambda: PlonkKzgSnark.prove_batch(ctx, pk1, tables1, [c1.pub_inputs] * 3, bls3, link_hints=True), 1),
        ("witness_batch", lambda p: p.submit_prove_witness_batch(pk1, [c1.witness] * 3, bls3, link_hints=True),
         lambda: PlonkKzgSnark.prove_witness_batch(ctx, pk1, [c1.witness] * 3, bls3, link_hints=True), 1),
        ("link", lambda p: p.submit_link(s.bases, e.hints[a], e.hints[b], lay),
         lambda: link_proofs(ctx, s.bases, e.hints[a], e.hints[b], lay)[0], 1),
        ("link_batch", lambda p: p.submit_link_batch(s.bases, triples), lambda: link_proofs_batch(ctx, s.bases, triples), 1),
        ("bundle", lambda p: p.submit_bundle(s.bases, bundle_tables, s.links), bundle_bare, 3),
        ("bundle_witness", lambda p: p.submit_bundle_witness(s.bases, bundle_witness, s.links),
         lambda: bundle_bare() + ([e.pubs[j] for j in range(3)],), 3),
        ("settlement", lambda p: p.submit_settlement(s.bases, pk1, s.tables[1], c1.pub_inputs, bl[1], settle_links),
         lambda: PlonkKzgSnark.prove_settlement(ctx, s.bases, pk1, s.tables[1], c1.pub_inputs, bl[1], settle_links), 1),
        ("settlement_witness", lambda p: p.submit_settlement_witness(s.bases, pk1, c1.witness, bl[1], settle_links),
         lambda: PlonkKzgSnark.prove_settlement_witness(ctx, s.bases, pk1, c1.witness, bl[1], settle_links), 1),
        ("verify_each", lambda p: p.submit_verify(*vargs, combined=False, g2=g2),
         lambda: PlonkKzgSnark.verify_each(ctx, *vargs, g2=g2), 1),
        ("batch_verify", lambda p: p.submit_verify(*vargs, combined=True, g2=g2),
         lambda: PlonkKzgSnark.batch_verify(ctx, *vargs, g2=g2), 1),
    ]


def test_every_job_kind_on_the_express_worker(env):
    lib = _lib.load()
    pool = ProverPool(0, workers=1, express=1)
    try:
        assert pool.workers == 1 and pool.context(0) is not None
        with pytest.raises(IndexError):  # the express context is the pool's own
            pool.context(1)
        for name, submit, bare, n_jobs in kinds(env):
            blocker = env.block(pool)
            t = submit(pool)
            assert pool.stats()["queued"] == n_jobs, name
            assert pool.expedite(t) == n_jobs, name
            got, done_at, worker = pool.wait_info(t)
            _, blocker_done_at, bw = pool.wait_info(blocker)
            assert bw == 0 and done_at < blocker_done_at, name  # the blocker outlasted the job: no normal worker was free
            assert worker == EXPRESS, name
            assert as_bytes(got) == as_bytes(bare()), name
        # a second proof of one key on the express worker replays its captured graphs there
        c0 = env.s.circs[0]
        want = as_bytes(PlonkKzgSnark.prove_witness(env.ctx, env.s.pks[0], c0.witness, env.bl[2])[:1])
        for _ in range(2):
            blocker = env.block(pool)
            g0 = lib.b200_graph_launches()
            t = pool.submit_prove_witness(env.s.pks[0], c0.witness, env.bl[2])
            assert pool.expedite(t) == 1
            got, _, worker = pool.wait_info(t)
            assert worker == EXPRESS and as_bytes(got[:1]) == want
            pool.wait(blocker)
        assert lib.b200_graph_launches() > g0
    finally:
        pool.close()


def test_expedite_order_without_express_workers(env):
    pool = ProverPool(0, workers=1)
    try:
        c0 = env.s.circs[0]
        blocker = env.block(pool)
        names = "ABCDEFGH"
        tickets = {n: pool.submit_prove_witness(env.s.pks[0], c0.witness, synth.splitmix_blinders(7600 + i))
                   for i, n in enumerate(names)}
        assert pool.stats()["queued"] == 8
        assert pool.expedite(tickets["H"]) == 1 and pool.expedite(tickets["G"]) == 1
        assert pool.stats()["queued"] == 8  # both queues
        _, first, w = pool.wait_info(blocker)
        assert w == 0
        done = {n: pool.wait_info(t) for n, t in tickets.items()}
        order = sorted(names, key=lambda n: done[n][1])
        assert order == list("HGABCDEF"), order
        assert [done[n][1] for n in order] == list(range(first + 1, first + 9))
        assert all(w == 0 for _, _, w in done.values())
    finally:
        pool.close()


def test_refusals_and_no_ops(env):
    lib = _lib.load()
    pool = ProverPool(0, workers=1, express=1)
    try:
        c0 = env.s.circs[0]
        with pytest.raises(_lib.B200Error) as err:  # never handed out
            pool.expedite(1 << 40)
        assert err.value.code == INVALID
        with pytest.raises(_lib.B200Error) as err:
            pool.wait_info(1 << 40)
        assert err.value.code == INVALID
        blocker = env.block(pool)
        assert pool.expedite(blocker) == 0  # running
        t = pool.submit_prove_witness(env.s.pks[0], c0.witness, env.bl[0])
        assert pool.expedite(t) == 1 and pool.expedite(t) == 0  # a second expedite moves nothing
        pool.wait(t)
        pool.wait(blocker)
        t = pool.submit_prove_witness(env.s.pks[0], c0.witness, env.bl[0])
        while pool.stats()["completed"] < pool.stats()["submitted"]:
            time.sleep(0.0005)
        assert pool.expedite(t) == 0  # finished, not yet waited for
        pool.wait(t)
        for call in (pool.expedite, pool.wait_info):  # waited for
            with pytest.raises(_lib.B200Error) as err:
                call(t)
            assert err.value.code == INVALID
        moved = C.c_size_t(5)
        assert lib.b200_pool_expedite(pool._h, 0, C.byref(moved)) == INVALID
        assert lib.b200_pool_expedite(pool._h, 1, None) == INVALID and moved.value == 5
        assert lib.b200_pool_wait_info(pool._h, 1, None) == INVALID
    finally:
        pool.close()
    h = C.c_void_p()
    for n, x in ((0, 0), (65, 0), (1, 65)):
        assert lib.b200_pool_create_express(0, n, x, C.byref(h)) == INVALID and not h.value
    devs = (C.c_int * 2)(0, 0)
    assert lib.b200_box_create_express(devs, 2, 1, 65, C.byref(h)) == INVALID and not h.value
    assert lib.b200_box_create_express(devs, 2, 0, 1, C.byref(h)) == INVALID and not h.value


@pytest.mark.parametrize("mode", [None, "0", "1"])
def test_stream_priority_modes(env, monkeypatch, mode):
    if mode is None:
        monkeypatch.delenv("B200_STREAM_PRIORITIES", raising=False)
    else:
        monkeypatch.setenv("B200_STREAM_PRIORITIES", mode)
    c0, pk0 = env.s.circs[0], env.s.pks[0]
    want = [as_bytes((lambda r: (r[0], r[1].linking_wire_poly))(PlonkKzgSnark.prove_witness(env.ctx, pk0, c0.witness, env.bl[i])))
            for i in range(3)]
    pool = ProverPool(0, workers=1, express=1)
    try:
        for i in range(3):  # eager, captured, replayed
            blocker = env.block(pool)
            t = pool.submit_prove_witness(pk0, c0.witness, env.bl[i], with_link_poly=True)
            assert pool.expedite(t) == 1
            (proof, poly, _), _, worker = pool.wait_info(t)
            assert worker == EXPRESS and as_bytes((proof, poly)) == want[i], i
            pool.wait(blocker)
    finally:
        pool.close()


def _pool_view(lib, handle):
    """A ProverPool over a box's device pool, which the box owns: closing the view leaves the pool alone."""
    p = ProverPool.__new__(ProverPool)
    p._lib, p._h, p.device, p._jobs, p._borrowed = lib, C.c_void_p(handle), 0, {}, []
    p.close = lambda: None
    return p


def test_box_expedite(env, oracle, pyoracle):
    lib = _lib.load()
    c0 = env.s.circs[0]
    box = ProverBox([0, 0], workers_per_device=1, express_per_device=1)
    try:
        tau = oracle.int_to_limbs(pyoracle.to_mont(TAU % pyoracle.R, pyoracle.R))
        srs = box.load_srs(oracle.srs_from_tau(tau, c0.n + 3))
        pk = box.preprocess_wiring(srs, c0.log_n, c0.num_inputs, c0.selectors, c0.wire_vars, c0.num_vars, c0.k)
        views = [_pool_view(lib, lib.b200_box_pool(box._h, i)) for i in range(2)]
        blockers = [env.block(v) for v in views]  # both entries busy: the job goes to entry 0 and waits there
        t = box.submit_prove_witness(pk, c0.witness, env.bl[1], with_link_poly=True)
        assert box.ticket_device(t) == 0
        assert box.expedite(t) == 1
        (proof, poly, pub), _, worker = box.wait_info(t)
        assert worker == EXPRESS
        want = PlonkKzgSnark.prove_witness(env.ctx, env.s.pks[0], c0.witness, env.bl[1])
        assert as_bytes((proof, poly, pub)) == as_bytes((want[0], want[1].linking_wire_poly, want[2]))
        for v, b in zip(views, blockers):
            v.wait(b)
        for bad in ((7 << 48) | 1, 1 << 40):  # a device index outside the box; a ticket entry 0 never handed out
            for call in (box.expedite, box.wait_info):
                with pytest.raises(_lib.B200Error) as err:
                    call(bad)
                assert err.value.code == INVALID
        box.free_pk(pk)
        box.free_srs(srs)
    finally:
        box.close()


@pytest.mark.parametrize("flow", ["private_match_flow", "intent_only_flow"])
def test_service_expedites_settlements(srs_2_16, srs_2_16_g2, flow):
    """The service flows over a pool with an express worker and `expedite_settlements`: every proof and link proof
    verifies, as on a plain pool."""
    import renegade_b200 as rb
    import service_flows
    from host_circuits import service_routes
    from renegade_b200 import circuit_types as ct
    from renegade_b200 import service as sv
    h, tau_h = srs_2_16_g2
    pool = ProverPool(0, workers=2, express=1)
    ctx = pool.context(0)
    params = rb.parse_ptau_file(ctx, srs_2_16, count=(1 << 14) + 3)
    ct.set_system_srs(ctx, params.powers_of_g, h, tau_h, pool=pool)
    service = sv.ProverService(service_routes.routes(), password="pw", pool=pool, expedite_settlements=True)
    server = service.make_server("127.0.0.1", 0)
    threading.Thread(target=server.serve_forever, daemon=True).start()
    try:
        client = sv.ProofServiceClient(f"http://127.0.0.1:{server.server_address[1]}", "pw")
        getattr(service_flows, flow)(client, service, srs_2_16_g2)
    finally:
        server.shutdown()
        server.server_close()
        ct.clear_key_cache()
        pool.close()
