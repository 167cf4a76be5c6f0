"""Cancellation of pool and box jobs (include/b200cancel.h).

A pool of one normal worker decides by submit order, not by timing, which job runs and which wait: a long blocker (a
witness batch of a 2^14 circuit, from test_gpu_express) runs while the jobs under test sit in the queue behind it.
Queued jobs of every kind are dropped without running (their output buffers keep a sentinel written after submit);
running jobs stop at an abort point or finish with their true status and bytes; a worker's context is as good after an
abort as before; `cancel_all` then `close` returns without running the queue."""
import ctypes as C
import threading
import time

import pytest

from renegade_b200 import _lib, synth
from renegade_b200.backend import B200Proof, PlonkKzgSnark, ProverBox, ProverPool, link_proofs
from test_gpu_express import Env, _pool_view, as_bytes, kinds

pytestmark = pytest.mark.gpu
OK, INVALID, CANCELLED = _lib.B200_OK, _lib.B200_ERR_INVALID, _lib.B200_ERR_CANCELLED
SENTINEL = 0xA5


@pytest.fixture(scope="module")
def env(ctx, oracle, pyoracle, srs_2_16_g2):
    e = Env(ctx, oracle, pyoracle, srs_2_16_g2)
    yield e
    e.free()


def _ctypes_in(obj, seen=None, out=None):
    """Every ctypes buffer a ticket holds (its held objects and the closures of its finish): the outputs the job writes,
    and input records the pool copied at submit, which the job no longer reads."""
    seen, out = (set(), []) if seen is None else (seen, out)
    if id(obj) in seen:
        return out
    seen.add(id(obj))
    if isinstance(obj, (C.Structure, C.Array)) or (isinstance(obj, C._SimpleCData) and not isinstance(obj, (C.c_void_p, C.c_char_p))):
        out.append(obj)
    elif isinstance(obj, (tuple, list)):
        for x in obj:
            _ctypes_in(x, seen, out)
    elif isinstance(obj, dict):
        for x in obj.values():
            _ctypes_in(x, seen, out)
    elif callable(obj) and getattr(obj, "__closure__", None):
        for cell in obj.__closure__:
            try:
                _ctypes_in(cell.cell_contents, seen, out)
            except ValueError:  # an empty cell
                pass
    return out


def _fill(bufs):
    for b in bufs:
        C.memset(C.addressof(b), SENTINEL, C.sizeof(b))


def _untouched(bufs):
    return all(C.string_at(C.addressof(b), C.sizeof(b)) == bytes([SENTINEL]) * C.sizeof(b) for b in bufs)


def _code(call, *args):
    """The error code `call` raises, or OK with its result."""
    try:
        return OK, call(*args)
    except _lib.B200Error as e:
        return e.code, None


def _started(pool, queued=0):
    while pool.stats()["queued"] > queued:
        time.sleep(0.0002)


def test_queued_jobs_of_every_kind_are_dropped(env):
    """Each kind queued behind the running blocker: cancel drops its jobs, its wait is B200_ERR_CANCELLED, its buffers
    keep the sentinel; the blocker's bytes are the bare context's."""
    pool = ProverPool(0, workers=1)
    try:
        blocker = env.block(pool)
        st0 = pool.stats()
        dropped_total = 0
        for name, submit, _, n_jobs in kinds(env):
            t = submit(pool)
            bufs = _ctypes_in(pool._jobs[t])
            assert bufs, name
            _fill(bufs)  # the job is queued behind the blocker: nothing writes these unless it runs
            assert pool.stats()["queued"] == n_jobs, name
            assert pool.cancel(t) == n_jobs, name
            assert pool.stats()["queued"] == 0, name
            assert pool.cancel(t) == 0, name  # twice is harmless
            assert _untouched(bufs), name
            code, _ = _code(pool.wait, t)
            assert code == CANCELLED, name
            dropped_total += n_jobs
        st = pool.stats()
        assert st["submitted"] - st0["submitted"] == dropped_total
        assert st["failed"] - st0["failed"] == dropped_total  # a dropped job counts as completed and failed
        got = pool.wait(blocker)
        bc = env.blocker_circ
        want = PlonkKzgSnark.prove_witness_batch(env.ctx, env.blocker_pk, [bc.witness] * len(env.blocker_bl), env.blocker_bl)
        assert as_bytes(got) == as_bytes(want)
        st = pool.stats()
        assert st["submitted"] == st["completed"] and st["queued"] == 0
    finally:
        pool.close()


@pytest.mark.parametrize("express", [0, 1])
def test_expedited_jobs_are_dropped_from_the_express_queue(env, express):
    pool = ProverPool(0, workers=1, express=express)
    try:
        blockers = [env.block(pool)]
        if express:  # the express worker busy too, so that the expedited job waits in the express queue
            t = pool.submit_prove_witness_batch(env.blocker_pk, [env.blocker_circ.witness] * 32, env.blocker_bl[:32])
            assert pool.expedite(t) == 1
            _started(pool)
            blockers.append(t)
        c0 = env.s.circs[0]
        keep = pool.submit_prove_witness(env.s.pks[0], c0.witness, env.bl[0])
        t = pool.submit_prove_witness(env.s.pks[0], c0.witness, env.bl[1])
        bundle = pool.submit_bundle_witness(env.s.bases, [(pk, c.witness, b) for pk, c, b in zip(env.s.pks, env.s.circs, env.bl)],
                                            env.s.links)
        assert pool.expedite(t) == 1 and pool.expedite(bundle) == 3
        assert pool.stats()["queued"] == 5
        assert pool.cancel(t) == 1 and pool.cancel(bundle) == 3
        assert pool.stats()["queued"] == 1  # the normal queue's job stays
        for x in (t, bundle):
            assert _code(pool.wait, x)[0] == CANCELLED
        want = PlonkKzgSnark.prove_witness(env.ctx, env.s.pks[0], c0.witness, env.bl[0])
        assert as_bytes(pool.wait(keep)[:1]) == as_bytes(want[:1])
        for b in blockers:
            pool.wait(b)
    finally:
        pool.close()


def _tampered(proof):
    bad = B200Proof.from_buffer_copy(proof)
    bad.wires_evals[0][0] ^= 1
    return bad


def test_running_combined_verify_stops_at_a_bisection_step(env):
    """k = 4096 items, every other one tampered: the combined job bisects for a long time; cancelled once it runs, it
    returns B200_ERR_CANCELLED long before the uncancelled run, whose verdicts are the bare context's."""
    k = 4096
    js = [i % 3 for i in range(k)]
    vks = [env.vks[j] for j in js]
    pubs = [env.pubs[j] for j in js]
    proofs = [env.proofs[j] if i % 2 == 0 else _tampered(env.proofs[j]) for i, j in enumerate(js)]
    g2 = (env.h, env.tau_h)
    pool = ProverPool(0, workers=1)
    try:
        t0 = time.perf_counter()
        t = pool.submit_verify(vks, pubs, proofs, combined=True, g2=g2)
        _started(pool)
        time.sleep(0.5)
        pool.cancel(t)
        code, res = _code(pool.wait, t)
        cancelled_s = time.perf_counter() - t0
        assert code in (CANCELLED, OK)
        t0 = time.perf_counter()
        full = pool.wait(pool.submit_verify(vks, pubs, proofs, combined=True, g2=g2))
        full_s = time.perf_counter() - t0
        assert full == (False, [i % 2 == 0 for i in range(k)])
        if code == OK:
            assert res == full
        print(f"\ncombined verify, k = {k}, half tampered: cancelled after 0.5 s of running -> returned in "
              f"{cancelled_s:.2f} s ({'cancelled' if code == CANCELLED else 'finished first'}); uncancelled {full_s:.2f} s")
        assert code == CANCELLED and cancelled_s < full_s / 2
        # the worker's context verifies as the bare context does after the abort
        items = [(env.vks[j], env.pubs[j], env.proofs[j]) for j in range(3)]
        assert pool.wait(pool.submit_verify(*map(list, zip(*items)), combined=True, g2=g2)) == (True, [True] * 3)
    finally:
        pool.close()


def test_running_prove_batch_stops_between_chunks(env, monkeypatch):
    monkeypatch.setenv("B200_PROVE_BATCH_CHUNK", "4")
    c1, pk1 = env.s.circs[1], env.s.pks[1]
    k = 64
    bls = [synth.splitmix_blinders(8100 + i) for i in range(k)]
    pool = ProverPool(0, workers=1)
    try:
        t = pool.submit_prove_witness_batch(pk1, [c1.witness] * k, bls)
        _started(pool)
        assert pool.cancel(t) == 0  # running: nothing to drop
        code, res = _code(pool.wait, t)
        want = PlonkKzgSnark.prove_witness_batch(env.ctx, pk1, [c1.witness] * k, bls)
        assert code == CANCELLED or as_bytes(res) == as_bytes(want)
        print(f"\nprove batch of {k} in chunks of 4: {'cancelled' if code == CANCELLED else 'finished first'}")
        _context_reused(env, pool)
    finally:
        pool.close()


def test_running_bundle_forks_no_links(env):
    """A bundle cancelled in its proof phase (its first proof, of the 2^14 key, running): its queued proofs are dropped,
    its ticket is B200_ERR_CANCELLED, and none of its link jobs is forked."""
    pool = ProverPool(0, workers=1)
    try:
        st0 = pool.stats()
        proofs = [(env.blocker_pk, env.blocker_circ.witness, env.blocker_bl[0])] + \
                 [(pk, c.witness, b) for pk, c, b in zip(env.s.pks, env.s.circs, env.bl)]
        links = [(a + 1, b + 1, lay) for a, b, lay in env.s.links]
        t = pool.submit_bundle_witness(env.s.bases, proofs, links)
        _started(pool, queued=3)  # the first proof runs, three wait
        assert pool.cancel(t) in (2, 3)  # 2: the first proof finished meanwhile and the second started
        assert _code(pool.wait, t)[0] == CANCELLED  # a cancelled bundle that had not finished
        pool.wait_all()
        st = pool.stats()
        assert st["submitted"] - st0["submitted"] == 4  # its proofs only: no link job was forked
        assert st["submitted"] == st["completed"] and st["queued"] == 0
        _context_reused(env, pool)
    finally:
        pool.close()


def _context_reused(env, pool):
    """After an abort, the worker's next proof, link proof and verification job give the bare context's bytes and verdicts,
    and a warm proof is 7 graph submissions."""
    lib = _lib.load()
    c0, pk0 = env.s.circs[0], env.s.pks[0]
    want = as_bytes(PlonkKzgSnark.prove_witness(env.ctx, pk0, c0.witness, env.bl[2])[:1])
    for i in range(3):  # eager or captured, then replayed
        g0 = lib.b200_graph_launches()
        assert as_bytes(pool.wait(pool.submit_prove_witness(pk0, c0.witness, env.bl[2]))[:1]) == want
        graphs = lib.b200_graph_launches() - g0
    assert graphs == 7
    a, b, lay = env.s.links[0]
    assert as_bytes(pool.wait(pool.submit_link(env.s.bases, env.hints[a], env.hints[b], lay))) == \
        as_bytes(link_proofs(env.ctx, env.s.bases, env.hints[a], env.hints[b], lay)[0])
    items = [(env.vks[j], env.pubs[j], env.proofs[j]) for j in range(3)]
    assert pool.wait(pool.submit_verify(*map(list, zip(*items)), g2=(env.h, env.tau_h))) == [True] * 3


def test_abort_while_capturing_drops_the_partial_graph_set(ctx, oracle, pyoracle):
    """The second proof of a key on a context captures its graphs; cancelled while it runs, the next proofs capture
    again and keep their bytes, and a warm proof is 7 graph submissions.  A 2^16 key, so that the proof is still running
    when the cancel lands."""
    from test_gpu_prove_witness import load_srs
    lib = _lib.load()
    c = synth.synth_circuit(16, num_inputs=2, seed=8500)
    bases = load_srs(ctx, oracle, pyoracle, c.n)
    pk = PlonkKzgSnark.preprocess_wiring(ctx, bases, c.log_n, c.num_inputs, c.selectors, c.wire_vars, c.num_vars, c.k)
    bl = [synth.splitmix_blinders(8600 + i) for i in range(4)]
    want = [as_bytes(PlonkKzgSnark.prove_witness(ctx, pk, c.witness, bl[i])[:1]) for i in range(4)]
    outcomes = []
    try:
        for _ in range(3):  # the cancel may still land after the proof's last abort point
            pool = ProverPool(0, workers=1)
            try:
                assert as_bytes(pool.wait(pool.submit_prove_witness(pk, c.witness, bl[0]))[:1]) == want[0]  # eager
                t = pool.submit_prove_witness(pk, c.witness, bl[1])  # the capturing proof
                _started(pool)
                pool.cancel(t)
                code, res = _code(pool.wait, t)
                outcomes.append(code)
                if code == OK:
                    assert as_bytes(res[:1]) == want[1]
                for i in (2, 3):  # captured again (or replayed), then replayed
                    g0 = lib.b200_graph_launches()
                    assert as_bytes(pool.wait(pool.submit_prove_witness(pk, c.witness, bl[i]))[:1]) == want[i]
                    assert lib.b200_graph_launches() - g0 == 7
            finally:
                pool.close()
            if code == CANCELLED:
                break
    finally:
        pk.free()
        bases.free()
    print(f"\ncapturing proof cancelled while running: outcomes {outcomes}")
    assert CANCELLED in outcomes


def test_finished_tickets_and_refusals(env):
    lib = _lib.load()
    c0, pk0 = env.s.circs[0], env.s.pks[0]
    pool = ProverPool(0, workers=1)
    try:
        h = pool._h
        dropped = C.c_size_t(77)
        assert lib.b200_pool_cancel(h, 1, None) == INVALID
        assert lib.b200_pool_cancel_all(h, None) == INVALID
        assert lib.b200_pool_cancel(h, 0, C.byref(dropped)) == INVALID
        assert lib.b200_pool_cancel(h, 1, C.byref(dropped)) == INVALID and b"unknown ticket" in lib.b200_last_error()
        assert dropped.value == 77
        assert pool.cancel_all() == 0  # nothing held
        t = pool.submit_prove_witness(pk0, c0.witness, env.bl[0])
        while pool.stats()["completed"] < pool.stats()["submitted"]:
            time.sleep(0.0005)
        assert pool.cancel(t) == 0 and pool.cancel(t) == 0  # finished, not yet waited for
        want = PlonkKzgSnark.prove_witness(env.ctx, pk0, c0.witness, env.bl[0])
        assert as_bytes(pool.wait(t)[:1]) == as_bytes(want[:1])  # its real result
        with pytest.raises(_lib.B200Error) as err:  # waited for
            pool.cancel(t)
        assert err.value.code == INVALID
        with pytest.raises(_lib.B200Error) as err:  # never handed out
            pool.cancel(1 << 40)
        assert err.value.code == INVALID
    finally:
        pool.close()


def _cancel_all_then_destroy(env, jobs, submit, n):
    """n proofs queued behind the blocker; cancel_all, every wait, then destroy: at most the running job completes."""
    blocker = env.block(jobs)
    c0, pk0 = env.s.circs[0], env.s.pks[0]
    tickets = [blocker] + [submit(pk0, c0.witness, synth.splitmix_blinders(8200 + i)) for i in range(n)]
    dropped = jobs.cancel_all()
    assert dropped == n
    codes = [_code(jobs.wait, t)[0] for t in tickets]
    assert codes.count(CANCELLED) >= n and set(codes) <= {OK, CANCELLED}
    return codes


def test_cancel_all_then_destroy(env):
    pool = ProverPool(0, workers=1)
    st0 = pool.stats()
    codes = _cancel_all_then_destroy(env, pool, pool.submit_prove_witness, 40)
    st = pool.stats()
    assert st["submitted"] == st["completed"] and st["queued"] == 0
    assert st["failed"] - st0["failed"] == codes.count(CANCELLED)
    # submits after cancel_all run as usual
    c0, pk0 = env.s.circs[0], env.s.pks[0]
    t = pool.submit_prove_witness(pk0, c0.witness, env.bl[0])
    assert as_bytes(pool.wait(t)[:1]) == as_bytes(PlonkKzgSnark.prove_witness(env.ctx, pk0, c0.witness, env.bl[0])[:1])
    # a deep queue, then cancel_all and destroy without waiting: the destroy does not run the queue
    env.block(pool)
    for i in range(40):
        pool.submit_prove_witness(pk0, c0.witness, synth.splitmix_blinders(8300 + i))
    t0 = time.perf_counter()
    assert pool.cancel_all() == 40
    pool.close()
    print(f"\ncancel_all + destroy with 40 queued behind a running 2^14 batch: {time.perf_counter() - t0:.3f} s")


def test_box_cancel(env, oracle, pyoracle):
    from test_gpu_prove_witness import TAU
    lib = _lib.load()
    c0 = env.s.circs[0]
    box = ProverBox([0], workers_per_device=1)
    try:
        tau = oracle.int_to_limbs(pyoracle.to_mont(TAU % pyoracle.R, pyoracle.R))
        srs = box.load_srs(oracle.srs_from_tau(tau, c0.n + 3))
        pk = box.preprocess_wiring(srs, c0.log_n, c0.num_inputs, c0.selectors, c0.wire_vars, c0.num_vars, c0.k)
        view = _pool_view(lib, lib.b200_box_pool(box._h, 0))
        blocker = env.block(view)
        t = box.submit_prove_witness(pk, c0.witness, env.bl[1])
        keep = box.submit_prove_witness(pk, c0.witness, env.bl[2])
        assert box.ticket_device(t) == 0
        assert box.cancel(t) == 1 and box.cancel(t) == 0
        assert _code(box.wait, t)[0] == CANCELLED
        want = PlonkKzgSnark.prove_witness(env.ctx, env.s.pks[0], c0.witness, env.bl[2])
        assert as_bytes(box.wait(keep)[:1]) == as_bytes(want[:1])
        view.wait(blocker)
        for bad in ((7 << 48) | 1, 1 << 40):  # a device index outside the box; a ticket never handed out
            with pytest.raises(_lib.B200Error) as err:
                box.cancel(bad)
            assert err.value.code == INVALID
        # cancel_all on a one-device box, then the stats of its pool
        tickets = [box.submit_prove_witness(pk, c0.witness, synth.splitmix_blinders(8400 + i)) for i in range(8)]
        box.cancel_all()
        codes = [_code(box.wait, x)[0] for x in tickets]
        assert set(codes) <= {OK, CANCELLED} and codes.count(CANCELLED) >= 7
        st = view.stats()
        assert st["submitted"] == st["completed"] and st["queued"] == 0
        box.free_pk(pk)
        box.free_srs(srs)
    finally:
        box.close()


def test_service_shutdown_under_load(srs_2_16, srs_2_16_g2):
    """Requests in flight when the service shuts down are answered (200, or 500 for a cancelled proof); none hangs, and
    no request thread is left behind."""
    import renegade_b200 as rb
    from host_circuits import service_routes
    from host_circuits import valid_balance_create as vbc
    from renegade_b200 import circuit_types as ct
    from renegade_b200 import service as sv
    threads_before = threading.active_count()
    h, tau_h = srs_2_16_g2
    pool = ProverPool(0, workers=2)
    ctx = pool.context(0)
    params = rb.parse_ptau_file(ctx, srs_2_16, count=(1 << 14) + 3)
    ct.set_system_srs(ctx, params.powers_of_g, h, tau_h, pool=pool)
    service = sv.ProverService(service_routes.routes(), password="pw", pool=pool)
    server = service.make_server("127.0.0.1", 0)
    serving = threading.Thread(target=server.serve_forever)
    serving.start()
    n = 16
    answers = [None] * n
    try:
        client = sv.ProofServiceClient(f"http://127.0.0.1:{server.server_address[1]}", "pw")
        w, s = vbc.create_witness_statement(21)
        body = {"statement": sv.to_json(s), "witness": sv.to_json(w)}
        assert client.send_request("/prove-valid-balance-create", body)[0] == 200  # keys made, service warm

        def ask(i):
            answers[i] = client.send_request("/prove-valid-balance-create", body)[0]
        askers = [threading.Thread(target=ask, args=(i,)) for i in range(n)]
        for a in askers:
            a.start()
        while service.stats["requests"] < n + 1:  # every request is in
            time.sleep(0.001)
        t0 = time.perf_counter()
        service.shutdown(server)
        for a in askers:
            a.join(timeout=60)
        assert not any(a.is_alive() for a in askers), "a request hung"
        print(f"\nservice shutdown with {n} requests in flight: {time.perf_counter() - t0:.3f} s; answers {sorted(answers)}")
        assert all(code == 200 or 500 <= code < 600 for code in answers), answers
        assert pool._h is None  # the pool was released
    finally:
        if serving.is_alive():
            server.shutdown()
        serving.join(timeout=10)
        ct.clear_key_cache()
        pool.close()
    deadline = time.time() + 10  # the request threads end as their connections close
    while threading.active_count() > threads_before and time.time() < deadline:
        time.sleep(0.01)
    assert threading.active_count() <= threads_before
