"""GPU: the prover pool (b200_pool, the counterpart of the reference's `NativeProofManager` thread pool,
native_proof_manager.rs:138-201).  Proofs made by pool workers are byte-identical to the proofs of
the single-context call with the same witness and blinders (hence to the oracle's, which
test_gpu_plonk pins), whatever worker ran them and in whatever order they finished; a failing job
reports ITS status and message to the thread that waits for it and leaves the pool usable; link
jobs match the direct call."""
import ctypes as C
import threading

import numpy as np
import pytest

from renegade_b200 import synth
from renegade_b200._lib import B200Error
from renegade_b200.backend import B200Proof, GroupLayout, PlonkKzgSnark, ProverPool, link_proofs

pytestmark = pytest.mark.gpu

TAU = 0x0c1d2e3f405162738495a6b7c8d9eafb0c1d2e3f405162738495a6b7c8d9eafb


def make(ctx, oracle, pyoracle, log_n, seed, link=None):
    py = pyoracle
    circ = synth.synth_circuit(log_n, num_inputs=6, seed=seed, check=(log_n <= 10), link=link)
    tau = oracle.int_to_limbs(py.to_mont(TAU % py.R, py.R))
    srs = oracle.srs_from_tau(tau, (1 << log_n) + 3)
    return circ, tau, srs


def test_pool_proofs_equal_direct_proofs(ctx, oracle, pyoracle):
    log_n = 11
    circ, tau, srs = make(ctx, oracle, pyoracle, log_n, seed=21)
    pool = ProverPool(0, workers=4)
    try:
        assert pool.workers == 4
        setup_ctx = pool.context(0)
        bases = setup_ctx.load_bases(srs)
        pk = PlonkKzgSnark.preprocess(setup_ctx, bases, log_n, circ.num_inputs, circ.selectors, circ.perm, circ.k)
        wires = np.ascontiguousarray(circ.wires, dtype=np.uint64)
        blinders = [synth.splitmix_blinders(900 + i) for i in range(12)]
        tickets = [pool.submit_prove(pk, wires.ctypes.data, circ.pub_inputs, b, with_link_poly=(i % 3 == 0), keep=wires)
                   for i, b in enumerate(blinders)]
        # wait in reverse submission order: results are looked up by ticket, not by completion order
        got = {}
        for i in reversed(range(len(tickets))):
            got[i] = pool.wait(tickets[i])
        st = pool.stats()
        assert st == {"submitted": 12, "completed": 12, "failed": 0, "queued": 0}
        opk = {"selector_comms": pk.selector_comms, "sigma_comms": pk.sigma_comms}
        for i, b in enumerate(blinders):
            ref, hint = PlonkKzgSnark.prove_with_link_hint(ctx, pk, circ.wires, circ.pub_inputs, b)
            if i % 3 == 0:
                proof, link = got[i]
                assert (link == hint.linking_wire_poly).all()
            else:
                proof = got[i]
            assert bytes(proof) == bytes(ref), i
        assert oracle.plonk_verify_known_tau(log_n, circ.num_inputs, circ.k, opk, circ.pub_inputs,
                                             oracle.PlonkProof.from_buffer_copy(bytes(got[5])), tau)
        with pytest.raises(B200Error) as ei:  # a ticket is consumed by its wait
            pool.wait(tickets[0])
        assert ei.value.code == -1 and "already waited" in str(ei.value)
        pk.free()
    finally:
        pool.close()


def test_pool_failed_job_reports_its_error_and_pool_survives(ctx, oracle, pyoracle):
    log_n = 9
    circ, tau, srs = make(ctx, oracle, pyoracle, log_n, seed=22)
    pool = ProverPool(0, workers=2)
    try:
        c0 = pool.context(0)
        bases = c0.load_bases(srs)
        pk = PlonkKzgSnark.preprocess(c0, bases, log_n, circ.num_inputs, circ.selectors, circ.perm, circ.k)
        good = np.ascontiguousarray(circ.wires, dtype=np.uint64)
        bad = good.copy()
        bad[4, circ.num_inputs + 3] = bad[4, circ.num_inputs + 4]
        bl = synth.splitmix_blinders(7)
        t_good1 = pool.submit_prove(pk, good.ctypes.data, circ.pub_inputs, bl)
        t_bad = pool.submit_prove(pk, bad.ctypes.data, circ.pub_inputs, bl)
        t_good2 = pool.submit_prove(pk, good.ctypes.data, circ.pub_inputs, bl)
        with pytest.raises(B200Error) as ei:
            pool.wait(t_bad)
        assert ei.value.code == -7 and "WrongQuotientPolyDegree" in str(ei.value)
        p1, p2 = pool.wait(t_good1), pool.wait(t_good2)
        assert bytes(p1) == bytes(p2)
        assert pool.stats()["failed"] == 1
        # wait_all reports the oldest failure among the jobs nobody waited for
        pool.submit_prove(pk, good.ctypes.data, circ.pub_inputs, bl)
        pool.submit_prove(pk, bad.ctypes.data, circ.pub_inputs, bl)
        with pytest.raises(B200Error) as ei:
            pool.wait_all()
        assert ei.value.code == -7
        pool.wait_all()  # nothing pending, nothing failed since
        pk.free()
    finally:
        pool.close()


def test_pool_destroy_drains_the_queue_into_caller_buffers(ctx, oracle, pyoracle):
    """`b200_pool_destroy` finishes what is queued (the reference's proof manager answers every job it took off
    the queue): results land in the caller's buffers although nobody waited.  The jobs go through the C entry point,
    so the caller owns the proof structs and reads them after the destroy."""
    log_n = 9
    circ, tau, srs = make(ctx, oracle, pyoracle, log_n, seed=23)
    bases = ctx.load_bases(srs)  # keys made on another context of the device are usable by the workers
    pk = PlonkKzgSnark.preprocess(ctx, bases, log_n, circ.num_inputs, circ.selectors, circ.perm, circ.k)
    wires = np.ascontiguousarray(circ.wires, dtype=np.uint64)
    pub = np.ascontiguousarray(circ.pub_inputs, dtype=np.uint64)
    bl = synth.splitmix_blinders(77)
    ref, _ = PlonkKzgSnark.prove_with_link_hint(ctx, pk, circ.wires, circ.pub_inputs, bl)
    pool = ProverPool(0, workers=2)
    proofs = [B200Proof() for _ in range(8)]
    ticket = C.c_uint64()
    ptr = lambda a: a.ctypes.data_as(C.c_void_p)  # noqa: E731
    for p in proofs:
        assert pool._lib.b200_pool_submit_prove(pool._h, pk._h, ptr(wires), ptr(pub), circ.num_inputs, ptr(bl),
                                                C.byref(p), None, C.byref(ticket)) == 0
    assert pool.stats()["submitted"] == 8
    pool.close()
    for p in proofs:
        assert bytes(p) == bytes(ref)
    pk.free()


def test_pool_submit_from_many_threads_and_link_jobs(ctx, oracle, pyoracle):
    """Any thread may submit and wait (the reference's workers answer on per-job oneshot channels);
    the settlement bundle's link proofs are queued like the reference forks them
    (native_proof_manager.rs:726-782)."""
    layout = GroupLayout(alignment=7, offset=20, size=9)
    py = pyoracle
    vals = [(i * 0xD1B54A32D192ED03 + 99) % py.R for i in range(layout.size)]
    log_n = 10
    circ_a, tau, srs = make(ctx, oracle, pyoracle, log_n, seed=31, link=(layout.alignment, layout.offset, vals))
    circ_b, _, _ = make(ctx, oracle, pyoracle, log_n, seed=32, link=(layout.alignment, layout.offset, vals))
    pool = ProverPool(0, workers=3)
    try:
        c0 = pool.context(0)
        bases = c0.load_bases(srs)
        pks = [PlonkKzgSnark.preprocess(c0, bases, log_n, c.num_inputs, c.selectors, c.perm, c.k) for c in (circ_a, circ_b)]
        results, errors = {}, []

        def client(idx, circ, pk):
            try:
                w = np.ascontiguousarray(circ.wires, dtype=np.uint64)
                t = pool.submit_prove(pk, w.ctypes.data, circ.pub_inputs, synth.splitmix_blinders(40 + idx),
                                      with_link_poly=True, keep=w)
                results[idx] = pool.wait(t)
            except Exception as e:  # pragma: no cover
                errors.append(e)
        ths = [threading.Thread(target=client, args=(i, c, pk)) for i, (c, pk) in enumerate(zip((circ_a, circ_b), pks))]
        for t in ths:
            t.start()
        for t in ths:
            t.join()
        assert not errors, errors
        from renegade_b200.backend import LinkingHint
        hints = [LinkingHint(linking_wire_poly=results[i][1],
                             linking_wire_comm=np.array(results[i][0].wires_poly_comms[0], dtype=np.uint64)) for i in (0, 1)]
        tickets = [pool.submit_link(bases, hints[0], hints[1], layout) for _ in range(4)]
        lps = [pool.wait(t) for t in tickets]
        direct, _ = link_proofs(ctx, bases, hints[0], hints[1], layout)
        for lp in lps:
            assert bytes(lp) == bytes(direct)
        assert oracle.plonk_link_verify_known_tau(hints[0].linking_wire_comm, hints[1].linking_wire_comm, layout.alignment,
                                                  layout.offset, layout.size,
                                                  oracle.LinkProof.from_buffer_copy(bytes(lps[0])), tau)
        for pk in pks:
            pk.free()
    finally:
        pool.close()


def test_pool_bundle_one_ticket_for_proofs_and_links(ctx, oracle, pyoracle):
    """`b200_pool_submit_bundle`: three proofs and two link proofs (0 <-> 1 on one group, 2 <-> 1 on the same group) under
    ONE ticket, the link proofs forked inside the pool once the proofs are in (the settlement arms of
    `handle_proof_job`, native_proof_manager.rs:526-584, 726-782).  Everything equals what the single calls produce; a
    bundle with an unsatisfied proof reports that failure and forks no links; a bad submission is refused up front."""
    from renegade_b200._lib import B200Error
    from renegade_b200.backend import LinkingHint
    layout = GroupLayout(alignment=7, offset=20, size=9)
    py = pyoracle
    vals = [(i * 0xD1B54A32D192ED03 + 99) % py.R for i in range(layout.size)]
    sizes = (10, 11, 10)
    made = [make(ctx, oracle, pyoracle, lg, seed=51 + i, link=(layout.alignment, layout.offset, vals)) for i, lg in enumerate(sizes)]
    circs = [m[0] for m in made]
    tau, srs = made[1][1], made[1][2]          # the largest SRS serves all three
    pool = ProverPool(0, workers=3)
    try:
        c0 = pool.context(0)
        bases = c0.load_bases(srs)
        pks = [PlonkKzgSnark.preprocess(c0, bases, lg, c.num_inputs, c.selectors, c.perm, c.k) for lg, c in zip(sizes, circs)]
        wires = [np.ascontiguousarray(c.wires, dtype=np.uint64) for c in circs]
        bl = [synth.splitmix_blinders(60 + i) for i in range(3)]
        t = pool.submit_bundle(bases, [(pks[i], wires[i].ctypes.data, circs[i].pub_inputs, bl[i]) for i in range(3)],
                               [(0, 1, layout), (2, 1, layout)])
        proofs, polys, links = pool.wait(t)
        for i in range(3):
            single, hint = PlonkKzgSnark.prove_with_link_hint(c0, pks[i], circs[i].wires, circs[i].pub_inputs, bl[i])
            assert bytes(proofs[i]) == bytes(single) and (polys[i] == hint.linking_wire_poly).all()
        hints = [LinkingHint(linking_wire_poly=polys[i], linking_wire_comm=np.array(proofs[i].wires_poly_comms[0], dtype=np.uint64))
                 for i in range(3)]
        for (a, b), lp in zip(((0, 1), (2, 1)), links):
            direct, _ = link_proofs(ctx, bases, hints[a], hints[b], layout)
            assert bytes(lp) == bytes(direct)
            assert oracle.plonk_link_verify_known_tau(hints[a].linking_wire_comm, hints[b].linking_wire_comm, layout.alignment,
                                                      layout.offset, layout.size, oracle.LinkProof.from_buffer_copy(bytes(lp)), tau)
        # an unsatisfied witness in the bundle: the ticket reports it, the pool goes on
        bad = wires[2].copy()
        bad[0, 5, 0] ^= np.uint64(1)
        t = pool.submit_bundle(bases, [(pks[0], wires[0].ctypes.data, circs[0].pub_inputs, bl[0]),
                                       (pks[2], bad.ctypes.data, circs[2].pub_inputs, bl[2])], [(0, 1, layout)])
        with pytest.raises(B200Error) as err:
            pool.wait(t)
        assert err.value.code == -7
        with pytest.raises(B200Error):      # a link naming a proof that is not in the bundle
            pool.submit_bundle(bases, [(pks[0], wires[0].ctypes.data, circs[0].pub_inputs, bl[0])], [(0, 3, layout)])
        assert pool.stats()["queued"] == 0
        for pk in pks:
            pk.free()
    finally:
        pool.close()


def test_box_routes_jobs_over_devices_with_replicated_keys(ctx, oracle, pyoracle):
    """`b200_box`: a pool per device, SRS and keys replicated, jobs to the least-loaded device.  On a one-GPU box the two
    "devices" are the same GPU twice — the routing, replication and ticket logic are what is checked: every proof equals
    the single-context proof, both pools get work, the verifying key is the same on every device."""
    import torch
    from renegade_b200.backend import ProverBox
    devices = [0, 1] if torch.cuda.device_count() >= 2 else [0, 0]
    log_n = 11
    circ, tau, srs = make(ctx, oracle, pyoracle, log_n, seed=71)
    box = ProverBox(devices, workers_per_device=2)
    try:
        bsrs = box.load_srs(srs, check_on_curve=True)
        pk = box.preprocess(bsrs, log_n, circ.num_inputs, circ.selectors, circ.perm, circ.k)
        bases = ctx.load_bases(srs)
        spk = PlonkKzgSnark.preprocess(ctx, bases, log_n, circ.num_inputs, circ.selectors, circ.perm, circ.k)
        sel, sig = box.verifying_key(pk)
        assert (sel == spk.selector_comms).all() and (sig == spk.sigma_comms).all()
        wires = np.ascontiguousarray(circ.wires, dtype=np.uint64)
        bl = [synth.splitmix_blinders(700 + i) for i in range(12)]
        tickets = [box.submit_prove(pk, wires.ctypes.data, circ.pub_inputs, b, keep=wires) for b in bl]
        used = {box.ticket_device(t) for t in tickets}
        assert used == {0, 1}                               # 12 jobs over 2 x 2 workers: both pools took some
        for t, b in zip(tickets, bl):
            proof = box.wait(t)
            single, _ = PlonkKzgSnark.prove_with_link_hint(ctx, spk, circ.wires, circ.pub_inputs, b)
            assert bytes(proof) == bytes(single)
        with pytest.raises(B200Error):
            box.wait(tickets[0])                            # a ticket is consumed by its wait
        box.free_pk(pk)
        box.free_srs(bsrs)
        spk.free()
    finally:
        box.close()
