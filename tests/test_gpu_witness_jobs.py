"""Witness vectors for every job shape that takes wire tables: bundles (`b200_pool_submit_bundle_witness`), pool batch
jobs (`b200_pool_submit_prove_witness_batch`) and the box (`b200_box_preprocess_wiring`, `b200_box_submit_prove_witness`,
`b200_box_submit_bundle_witness`).  Every proof, link polynomial, public-input vector and link proof equals what the
table entry points and the single calls make from the same witness and blinders; failures are reported per ticket and
leave the pool usable; refusals queue nothing; bundle proofs replay their graphs like single proofs."""
import ctypes as C
import os
import subprocess
import threading

import numpy as np
import pytest

from renegade_b200 import _lib, synth
from renegade_b200.backend import (BundleLink, BundleWitness, GroupLayout, LinkingHint, PlonkKzgSnark, ProverBox,
                                   ProverPool, link_proofs)
from test_gpu_prove_witness import TAU, load_srs, unsatisfying
from test_prove_witness_cpu import expand, wiring_permutation

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INVALID, UNSAT = _lib.B200_ERR_INVALID, _lib.B200_ERR_UNSATISFIED


def tau_limbs(oracle, pyoracle):
    return oracle.int_to_limbs(pyoracle.to_mont(TAU % pyoracle.R, pyoracle.R))


def private_match():
    """The five statements of a private match and its four links, built as bench.py's private_match_bundle leg builds
    them: proof 0 PRIVATE SETTLEMENT (2^12), 1-2 INTENT AND BALANCE VALIDITY (2^14), 3-4 OUTPUT BALANCE VALIDITY (2^13);
    each link joins a validity proof to the settlement proof."""
    from host_circuits import intent_and_balance_validity as val
    from host_circuits import output_balance_validity as obv
    from host_circuits import private_settlement as ps
    parties, _ = ps.create_witness_statement(seed=61)
    validity = [val.create_witness_statement(seed=70 + i, intent=parties[i].intent, balance=parties[i].input_balance)
                for i in (0, 1)]
    out_validity = [obv.create_witness_statement(80 + i, parties[i].output_balance) for i in (0, 1)]
    parties, statement = ps.create_witness_statement(
        seed=61, linked=[(validity[i][0].new_amount_public_share, validity[i][0].post_match_balance_shares,
                          out_validity[i][0].post_match_balance_shares) for i in (0, 1)])
    settlement_cs = ps.IntentAndBalancePrivateSettlementCircuit.build(parties, statement)
    layouts = settlement_cs.get_circuit_layout()
    circs = [settlement_cs.finalize_for_arithmetization()] + \
            [val.IntentAndBalanceValidityCircuit.build(w, st, layouts).finalize_for_arithmetization() for w, st in validity] + \
            [obv.OutputBalanceValidityCircuit.build(w, st, layouts).finalize_for_arithmetization() for w, st in out_validity]
    lay = lambda g: GroupLayout(layouts[g].alignment, layouts[g].offset, layouts[g].size)  # noqa: E731
    links = [(1 + p, 0, lay(g)) for p, g in enumerate(ps.PARTY_LINKS)] + \
            [(3 + p, 0, lay(g)) for p, g in enumerate(ps.OUTPUT_LINKS)]
    return circs, links


def synthetic():
    """Three synthetic circuits (2^10, 2^11, 2^10) sharing one link group; links 0 <-> 1 and 2 <-> 1."""
    layout = GroupLayout(alignment=7, offset=20, size=9)
    vals = [(i * 0xD1B54A32D192ED03 + 99) % synth.R for i in range(layout.size)]
    circs = [synth.synth_circuit(lg, num_inputs=6, seed=51 + i, link=(layout.alignment, layout.offset, vals))
             for i, lg in enumerate((10, 11, 10))]
    return circs, [(0, 1, layout), (2, 1, layout)]


class Setup:
    """A bundle shape with its SRS and its keys from the wiring, made on the session context (workers use them too)."""

    def __init__(self, ctx, oracle, pyoracle, circs, links):
        self.circs, self.links = circs, links
        self.bases = load_srs(ctx, oracle, pyoracle, max(c.n for c in circs))
        self.pks = [PlonkKzgSnark.preprocess_wiring(ctx, self.bases, c.log_n, c.num_inputs, c.selectors, c.wire_vars,
                                                    c.num_vars, c.k) for c in circs]
        self.tables = [np.ascontiguousarray(expand(c)) for c in circs]

    def free(self):
        for pk in self.pks:
            pk.free()
        self.bases.free()


@pytest.fixture(scope="module")
def pool():
    p = ProverPool(0, workers=4)
    yield p
    p.close()


@pytest.fixture(scope="module", params=["private_match", "synthetic"])
def shape(request, ctx, oracle, pyoracle):
    s = Setup(ctx, oracle, pyoracle, *(private_match() if request.param == "private_match" else synthetic()))
    yield s
    s.free()


def blinders(base, k):
    return [synth.splitmix_blinders(base + i) for i in range(k)]


def as_bytes(res):
    """A bundle result as bytes: proofs, link polys, link proofs (and public inputs, for a witness bundle)."""
    return [[bytes(x) if not isinstance(x, np.ndarray) else x.tobytes() for x in part] for part in res]


def test_bundle_equals_tables_and_single_calls(ctx, oracle, pyoracle, pool, shape):
    s, bl = shape, blinders(8000, len(shape.circs))
    res = pool.wait(pool.submit_bundle_witness(s.bases, [(pk, c.witness, b) for pk, c, b in zip(s.pks, s.circs, bl)], s.links))
    proofs, polys, lps, pubs = res
    tables = pool.wait(pool.submit_bundle(s.bases, [(pk, w.ctypes.data, c.pub_inputs, b)
                                                   for pk, w, c, b in zip(s.pks, s.tables, s.circs, bl)], s.links))
    assert as_bytes(res)[:3] == as_bytes(tables)
    hints = []
    for j, (pk, c, b) in enumerate(zip(s.pks, s.circs, bl)):
        proof, hint, pub = PlonkKzgSnark.prove_witness(ctx, pk, c.witness, b)
        assert bytes(proofs[j]) == bytes(proof) and polys[j].tobytes() == hint.linking_wire_poly.tobytes(), j
        assert pubs[j].tobytes() == pub.tobytes() == np.ascontiguousarray(c.pub_inputs).tobytes(), j
        hints.append(LinkingHint(linking_wire_poly=polys[j], linking_wire_comm=np.array(proofs[j].wires_poly_comms[0],
                                                                                        dtype=np.uint64)))
    tau = tau_limbs(oracle, pyoracle)
    for (a, b, lay), lp in zip(s.links, lps):
        direct, _ = link_proofs(ctx, s.bases, hints[a], hints[b], lay)
        assert bytes(lp) == bytes(direct)
        assert oracle.plonk_link_verify_known_tau(hints[a].linking_wire_comm, hints[b].linking_wire_comm, lay.alignment,
                                                  lay.offset, lay.size, oracle.LinkProof.from_buffer_copy(bytes(lp)), tau)


@pytest.fixture(scope="module")
def small(ctx, oracle, pyoracle):
    s = Setup(ctx, oracle, pyoracle, *synthetic())
    yield s
    s.free()


def test_bundle_pointer_kinds(pool, small):
    """numpy, pinned host, device and device + 16 bytes witnesses in one bundle: the outputs do not change."""
    import torch
    s, bl = small, blinders(8100, 4)
    idx = [0, 1, 2, 0]  # proof 3 repeats circuit 0
    ref = pool.wait(pool.submit_bundle_witness(s.bases, [(s.pks[i], s.circs[i].witness, b) for i, b in zip(idx, bl)],
                                               s.links))
    w = [np.ascontiguousarray(s.circs[i].witness) for i in idx]
    pinned = torch.from_numpy(w[1].view(np.int64)).pin_memory()
    dev = torch.from_numpy(w[2].view(np.int64)).cuda()
    dev16 = torch.zeros(w[3].size + 2, dtype=torch.int64, device="cuda")
    dev16[2:] = torch.from_numpy(w[3].view(np.int64).reshape(-1)).cuda()
    torch.cuda.synchronize()
    ptrs = [w[0], pinned.data_ptr(), dev.data_ptr(), dev16.data_ptr() + 16]
    got = pool.wait(pool.submit_bundle_witness(s.bases, [(s.pks[i], p, b) for i, p, b in zip(idx, ptrs, bl)], s.links))
    assert as_bytes(got) == as_bytes(ref)


def test_bundle_failures(pool, small):
    s, bl = small, blinders(8200, 3)
    entries = [(pk, c.witness, b) for pk, c, b in zip(s.pks, s.circs, bl)]
    before = pool.stats()["submitted"]
    bad = list(entries)
    bad[2] = (s.pks[2], unsatisfying(s.circs[2]), bl[2])
    with pytest.raises(_lib.B200Error) as err:
        pool.wait(pool.submit_bundle_witness(s.bases, bad, s.links))
    assert err.value.code == UNSAT
    assert pool.stats()["submitted"] - before == 3  # the three proofs and no link job
    good = pool.wait(pool.submit_bundle_witness(s.bases, entries, s.links))  # the pool goes on
    assert len(good[2]) == 2
    # refusals at submit, straight through the C ABI: nothing queued, nothing counted
    lib, p = pool._lib, lambda a: a.ctypes.data_as(C.c_void_p)  # noqa: E731
    table_pk = PlonkKzgSnark.preprocess(pool.context(0), s.bases, s.circs[0].log_n, s.circs[0].num_inputs,
                                        s.circs[0].selectors, wiring_permutation(s.circs[0].wire_vars), s.circs[0].k)
    proofs = [_lib.STRUCTS["b200_proof"]() for _ in range(2)]
    polys = [np.zeros((c.n + 2, 4), dtype=np.uint64) for c in s.circs[:2]]
    wits = [np.ascontiguousarray(c.witness) for c in s.circs[:2]]
    lproof = _lib.STRUCTS["b200_link_proof"]()

    def arrays(pk0=None, wit0=True, poly1=True, link_b=1):
        arr = (BundleWitness * 2)()
        for i in range(2):
            arr[i] = BundleWitness(s.pks[i]._h, p(wits[i]), p(bl[i]), C.cast(C.pointer(proofs[i]), C.c_void_p),
                                   p(polys[i]), None)
        if pk0 is not None:
            arr[0].pk = pk0
        if not wit0:
            arr[0].witness = None
        if not poly1:
            arr[1].link_poly = None
        lay = s.links[0][2]
        link = (BundleLink * 1)(BundleLink(0, link_b, lay.alignment, lay.offset, lay.size, C.cast(C.pointer(lproof), C.c_void_p)))
        return arr, link

    st0, t = pool.stats(), C.c_uint64()
    for kw, msg in (({"wit0": False}, b"NULL"), ({"pk0": table_pk._h}, b"wiring"), ({"link_b": 2}, b"missing"),
                    ({"poly1": False}, b"link_poly")):
        arr, link = arrays(**kw)
        assert lib.b200_pool_submit_bundle_witness(pool._h, s.bases._h, arr, 2, link, 1, C.byref(t)) == INVALID, kw
        assert msg in lib.b200_last_error(), kw
    assert lib.b200_pool_submit_bundle_witness(pool._h, None, arrays()[0], 2, arrays()[1], 1, C.byref(t)) == INVALID
    assert pool.stats() == st0 and st0["queued"] == 0
    table_pk.free()


def test_pool_witness_batch_job(ctx, oracle, pyoracle, pool):
    circ = synth.synth_circuit(8, num_inputs=2, seed=8)
    bases = load_srs(ctx, oracle, pyoracle, circ.n)
    pk = PlonkKzgSnark.preprocess_wiring(ctx, bases, circ.log_n, circ.num_inputs, circ.selectors, circ.wire_vars,
                                         circ.num_vars, circ.k)
    bad = unsatisfying(circ)
    k = 65  # one past a 64-proof gather group
    wits = [bad if i in (0, 63, 64) else circ.witness for i in range(k)]
    bls = blinders(9000, k)
    want = PlonkKzgSnark.prove_witness_batch(ctx, pk, wits, bls, link_hints=True)
    got = pool.wait(pool.submit_prove_witness_batch(pk, wits, bls, link_hints=True))
    assert got[2] == want[2] and [i for i, st in enumerate(got[2]) if st] == [0, 63, 64]
    assert [bytes(x) for x in got[0]] == [bytes(x) for x in want[0]]
    assert [h and h.linking_wire_poly.tobytes() for h in got[1]] == [h and h.linking_wire_poly.tobytes() for h in want[1]]
    assert [x.tobytes() for x in got[3]] == [x.tobytes() for x in want[3]]
    pk.free()
    bases.free()


def test_pool_jobs_from_two_threads(ctx, pool, small):
    """Witness batch jobs from two threads, interleaved with single witness jobs and a table bundle: the same bytes."""
    s = small
    c, pk = s.circs[1], s.pks[1]
    bls = blinders(9500, 6)
    single = [bytes(PlonkKzgSnark.prove_witness(ctx, pk, c.witness, b)[0]) for b in bls]
    tb = [(q, w.ctypes.data, cc.pub_inputs, b) for q, w, cc, b in zip(s.pks, s.tables, s.circs, blinders(9600, 3))]
    bundle_ref = as_bytes(pool.wait(pool.submit_bundle(s.bases, tb, s.links)))
    results, errors = {}, []

    def client(tid):
        try:
            out = []
            for r in range(3):
                tks = [("batch", pool.submit_prove_witness_batch(pk, [c.witness] * 6, bls)),
                       ("single", pool.submit_prove_witness(pk, c.witness, bls[r])),
                       ("bundle", pool.submit_bundle(s.bases, tb, s.links))]
                out.append([(kind, pool.wait(t)) for kind, t in tks])
            results[tid] = out
        except Exception as e:  # pragma: no cover
            errors.append(e)
    ths = [threading.Thread(target=client, args=(i,)) for i in range(2)]
    for t in ths:
        t.start()
    for t in ths:
        t.join()
    assert not errors, errors
    for tid in (0, 1):
        for r, round_ in enumerate(results[tid]):
            (_, batch), (_, one), (_, bundle) = round_
            assert [bytes(x) for x in batch[0]] == single and batch[2] == [0] * 6
            assert bytes(one[0]) == single[r]
            assert as_bytes(bundle) == bundle_ref


def test_bundle_proofs_replay_their_graphs(ctx, oracle, pyoracle, small):
    """After one proof of each key on a worker, every proof of a witness bundle runs as 7 graph submissions."""
    s = small
    one = ProverPool(0, workers=1)
    try:
        for pk, c, b in zip(s.pks, s.circs, blinders(9700, 3)):
            one.wait(one.submit_prove_witness(pk, c.witness, b))
        entries = [(pk, c.witness, b) for pk, c, b in zip(s.pks, s.circs, blinders(9800, 3))]
        for _ in range(2):
            g0 = ctx.graph_launches()
            one.wait(one.submit_bundle_witness(s.bases, entries, []))
            assert ctx.graph_launches() - g0 == 3 * 7
    finally:
        one.close()


def box_devices():
    import torch
    return [0, 1] if torch.cuda.device_count() >= 2 else [0, 0]


def test_box_witness_jobs(ctx, oracle, pyoracle, small):
    import torch
    s, devices = small, box_devices()
    c = s.circs[1]
    srs = oracle.srs_from_tau(tau_limbs(oracle, pyoracle), max(cc.n for cc in s.circs) + 3)
    box, other = ProverBox(devices, workers_per_device=2), ProverBox(devices, workers_per_device=1)
    try:
        bsrs = box.load_srs(srs)
        bpks = [box.preprocess_wiring(bsrs, cc.log_n, cc.num_inputs, cc.selectors, cc.wire_vars, cc.num_vars, cc.k)
                for cc in s.circs]
        for bpk, pk in zip(bpks, s.pks):
            sel, sig = box.verifying_key(bpk)
            assert (sel == pk.selector_comms).all() and (sig == pk.sigma_comms).all()
        # twelve witness jobs use both pools; every proof is the single-context proof
        bls = blinders(9900, 12)
        tks = [box.submit_prove_witness(bpks[1], c.witness, b, with_link_poly=(i % 2 == 0)) for i, b in enumerate(bls)]
        assert {box.ticket_device(t) for t in tks} == {0, 1}
        for i, (t, b) in enumerate(zip(tks, bls)):
            out = box.wait(t)
            proof, hint, pub = PlonkKzgSnark.prove_witness(ctx, s.pks[1], c.witness, b)
            assert bytes(out[0]) == bytes(proof) and out[-1].tobytes() == pub.tobytes(), i
            if i % 2 == 0:
                assert out[1].tobytes() == hint.linking_wire_poly.tobytes()
        # a device-memory witness runs on the device that holds it
        dev = devices[-1]
        with torch.cuda.device(dev):
            d_w = torch.from_numpy(np.ascontiguousarray(c.witness).view(np.int64)).to(f"cuda:{dev}")
            torch.cuda.synchronize()
        for b in bls[:4]:
            t = box.submit_prove_witness(bpks[1], d_w.data_ptr(), b)
            assert devices[box.ticket_device(t)] == dev
            assert bytes(box.wait(t)[0]) == bytes(PlonkKzgSnark.prove_witness(ctx, s.pks[1], c.witness, b)[0])
        # bundles on the box equal the pool bundle, from tables and from witness vectors
        bb = blinders(9950, 3)
        pool = ProverPool(0, workers=2)
        try:
            want = as_bytes(pool.wait(pool.submit_bundle_witness(s.bases, [(pk, cc.witness, b) for pk, cc, b in
                                                                           zip(s.pks, s.circs, bb)], s.links)))
        finally:
            pool.close()
        got = box.wait(box.submit_bundle_witness(bsrs, [(q, cc.witness, b) for q, cc, b in zip(bpks, s.circs, bb)], s.links))
        assert as_bytes(got) == want
        got = box.wait(box.submit_bundle(bsrs, [(q, w.ctypes.data, cc.pub_inputs, b) for q, w, cc, b in
                                                zip(bpks, s.tables, s.circs, bb)], s.links))
        assert as_bytes(got) == want[:3]
        if devices == [0, 1]:  # device witnesses on two devices cannot make one bundle
            d0 = torch.from_numpy(np.ascontiguousarray(s.circs[0].witness).view(np.int64)).to("cuda:0")
            torch.cuda.synchronize()
            with pytest.raises(_lib.B200Error) as err:
                box.submit_bundle_witness(bsrs, [(bpks[0], d0.data_ptr(), bb[0]), (bpks[1], d_w.data_ptr(), bb[1])], [])
            assert err.value.code == INVALID and "two devices" in str(err.value)
        # a key from another box is refused, by the wrapper and by the library
        osrs = other.load_srs(srs)
        opk = other.preprocess_wiring(osrs, c.log_n, c.num_inputs, c.selectors, c.wire_vars, c.num_vars, c.k)
        with pytest.raises(_lib.B200Error):
            box.submit_prove_witness(opk, c.witness, bls[0])
        proof, wit, t = _lib.STRUCTS["b200_proof"](), np.ascontiguousarray(c.witness), C.c_uint64()
        p = lambda a: a.ctypes.data_as(C.c_void_p)  # noqa: E731
        assert box._lib.b200_box_submit_prove_witness(box._h, opk, p(wit), p(bls[0]), C.byref(proof), None, None,
                                                      C.byref(t)) == INVALID
        assert b"another box" in box._lib.b200_last_error()
        other.free_pk(opk)
        other.free_srs(osrs)
        for q in bpks:
            box.free_pk(q)
        box.free_srs(bsrs)
    finally:
        box.close()
        other.close()


def test_c_host_harness_witness_bundle(tmp_path, oracle, pyoracle):
    """examples/host_harness.c proves a witness bundle (2 proofs, 1 link) through a pool; its bytes are the oracle's."""
    py = pyoracle
    exe, src = os.path.join(ROOT, "examples", "host_harness"), os.path.join(ROOT, "examples", "host_harness.c")
    if not os.path.exists(exe) or os.path.getmtime(exe) < os.path.getmtime(src):
        subprocess.check_call(["gcc", "-O2", "-I" + os.path.join(ROOT, "include"), src, "-L" + os.path.join(ROOT, "renegade_b200"),
                               "-lb200prover", "-Wl,-rpath," + os.path.join(ROOT, "renegade_b200"), "-o", exe])
    log_n, n = 10, 1 << 10
    circ = synth.synth_circuit(log_n, num_inputs=4, seed=21, check=True)
    tau = oracle.int_to_limbs(py.to_mont(0x0123456789abcdef0fedcba9876543210011223344556677 % py.R, py.R))
    srs = oracle.srs_from_tau(tau, n + 3)
    bl = synth.splitmix_blinders(0xC)
    job = tmp_path / "job.bin"
    with open(job, "wb") as f:
        f.write(np.array([log_n, circ.num_inputs, n + 3], dtype=np.uint64).tobytes())
        for arr in (circ.k, circ.selectors, circ.perm, circ.wires, circ.pub_inputs, bl, srs):
            f.write(np.ascontiguousarray(arr, dtype=np.uint64).tobytes())
    r = subprocess.run([exe, str(job), str(tmp_path / "proof.bin"), str(tmp_path / "bundle.bin")], capture_output=True,
                       text=True, timeout=300)
    assert r.returncode == 0, r.stderr
    blob = open(tmp_path / "bundle.bin", "rb").read()
    assert len(blob) == 2 * 1152 + 128
    # the harness numbers one variable per cycle of the job's permutation, in the order the cycles are first met
    wire_vars, nv = np.full(5 * n, -1, dtype=np.int64), 0
    for q0 in range(5 * n):
        q = q0
        while wire_vars[q] < 0:
            wire_vars[q] = nv
            q = int(circ.perm[q])
        nv += wire_vars[q0] == nv
    opk = oracle.plonk_preprocess(log_n, circ.selectors, wiring_permutation(wire_vars.astype(np.uint32)), circ.k, srs)
    outs = []
    for b in (bl, np.ascontiguousarray(bl.reshape(17, 4)[::-1])):
        rc, oproof, _, olink = oracle.plonk_prove(log_n, circ.num_inputs, circ.k, opk, circ.wires, circ.pub_inputs, b, srs, True)
        assert rc == 0
        outs.append((oproof, olink))
    assert blob[:1152] == bytes(outs[0][0]) and blob[1152:2304] == bytes(outs[1][0])
    comms = [o[0].to_array()[:8].copy() for o in outs]
    rc, olp, _ = oracle.plonk_link(outs[0][1], outs[1][1], comms[0], comms[1], log_n, circ.num_inputs, 4, srs)
    assert rc == 0 and blob[2304:] == bytes(olp)
    assert oracle.plonk_link_verify_known_tau(comms[0], comms[1], log_n, circ.num_inputs, 4,
                                              oracle.LinkProof.from_buffer_copy(blob[2304:]), tau)
