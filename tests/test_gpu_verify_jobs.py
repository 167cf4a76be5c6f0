"""Verification jobs on a pool and a box (`b200_pool_submit_verify`, `b200_box_submit_verify`, `ProverPool.submit_verify`,
`ProverBox.submit_verify`): in both modes the verdicts and the combined answer equal the bare-context calls
(`b200_plonk_verify_each` / `b200_plonk_batch_verify`) on the same items; inputs may be freed or overwritten as soon as
the submit returns; verification jobs interleave with prove, bundle and settlement jobs without changing any proof's
bytes; refusals at submit queue nothing.

The items are gossip-shaped orders over the restated private-match statements (examples/host_circuits): the PRIVATE
SETTLEMENT (2^12), the INTENT AND BALANCE VALIDITY (2^14) and OUTPUT BALANCE VALIDITY (2^13) proofs and their link proofs,
plus a seeded share of the tamperings of tests/verify_mutations.py."""
import ctypes as C
import random
import threading

import numpy as np
import pytest

import verify_mutations as vm
from renegade_b200 import _lib
from renegade_b200.backend import (B200LinkProof, B200Proof, GroupLayout, PlonkKzgSnark, ProverBox, ProverPool,
                                   VerifyingKey, _VerifyBatch, link_proofs)
from test_gpu_witness_jobs import Setup, private_match

pytestmark = pytest.mark.gpu
OK, INVALID, NOT_ON_CURVE = _lib.B200_OK, _lib.B200_ERR_INVALID, _lib.B200_ERR_NOT_ON_CURVE
KINDS = ("eval_bit", "swap_comms", "pub_input", "off_curve", "encoding_ge_p", "link_layout")


class Env:
    """The private match proved on the session context: keys, proofs, hints, link proofs, verifying keys."""

    def __init__(self, ctx, oracle, pyoracle, g2):
        from renegade_b200 import synth
        self.s = Setup(ctx, oracle, pyoracle, *private_match())
        self.ctx, self.h, self.tau_h = ctx, g2[0], g2[1]
        self.bl = [synth.splitmix_blinders(6100 + j) for j in range(len(self.s.circs))]
        self.proofs, self.hints, self.pubs = [], [], []
        for pk, c, b in zip(self.s.pks, self.s.circs, self.bl):
            proof, hint, pub = PlonkKzgSnark.prove_witness(ctx, pk, c.witness, b)
            self.proofs.append(proof)
            self.hints.append(hint)
            self.pubs.append(pub)
        self.vks = [VerifyingKey.from_proving_key(pk, self.h, self.tau_h) for pk in self.s.pks]
        self.link_proofs = [link_proofs(ctx, self.s.bases, self.hints[a], self.hints[b], lay)[0] for a, b, lay in self.s.links]

    def order(self, i):
        """Order i: a validity proof, the settlement proof and the link proof between them."""
        a, b, lay = self.s.links[i % len(self.s.links)]
        proofs = [(self.vks[a], self.pubs[a], self.proofs[a]), (self.vks[b], self.pubs[b], self.proofs[b])]
        link = (self.hints[a].linking_wire_comm, self.hints[b].linking_wire_comm, self.link_proofs[i % len(self.s.links)], lay)
        return proofs, [link]

    def orders(self, k, seed=None, share=0.25):
        """k orders as one job's items; with a seed, a seeded share of the orders carry one tampering each."""
        proofs, links = [], []
        rnd = random.Random(seed)
        for i in range(k):
            ps, ls = self.order(i)
            if seed is not None and rnd.random() < share:
                kind = KINDS[rnd.randrange(len(KINDS))]
                if kind == "link_layout":
                    ls = [tamper_link(ls[0])]
                else:
                    j = rnd.randrange(2)
                    ps[j] = tamper_proof(ps[j], kind)
            proofs += ps
            links += ls
        return proofs, links

    def free(self):
        self.s.free()


def tamper_proof(item, kind):
    vk, pi, proof = item
    p = B200Proof.from_buffer_copy(bytes(proof))
    if kind == "eval_bit":
        p.wires_evals[3][0] ^= 1
    elif kind == "swap_comms":
        w0, w1 = list(p.wires_poly_comms[0]), list(p.wires_poly_comms[1])
        p.wires_poly_comms[0][:], p.wires_poly_comms[1][:] = w1, w0
    elif kind == "pub_input":
        pi = np.array(pi, dtype=np.uint64).copy()
        pi[0, 0] ^= np.uint64(1)
    elif kind == "off_curve":
        p.opening_proof[0] ^= 1
    elif kind == "encoding_ge_p":  # an evaluation v + r: the same residue, outside [0, r)
        v = vm.to_int(np.array(p.perm_next_eval, dtype=np.uint64))
        p.perm_next_eval[:] = [int(w) for w in vm.to_words(vm.out_of_field(v, vm.R)["plus_p"])]
    return vk, pi, p


def tamper_link(link):
    a, b, lp, lay = link
    return a, b, lp, GroupLayout(lay.alignment, lay.offset + 1, lay.size)


@pytest.fixture(scope="module")
def env(ctx, oracle, pyoracle, srs_2_16_g2):
    e = Env(ctx, oracle, pyoracle, srs_2_16_g2)
    yield e
    e.free()


@pytest.fixture(scope="module")
def pool():
    p = ProverPool(0, workers=4)
    yield p
    p.close()


@pytest.fixture(scope="module")
def box():
    b = ProverBox([0, 0], workers_per_device=2)  # two box entries on one device: routing still picks the least loaded
    yield b
    b.close()


def bare(e, proofs, links, combined):
    args = ([p[0] for p in proofs], [p[1] for p in proofs], [p[2] for p in proofs], links)
    if combined:
        return PlonkKzgSnark.batch_verify(e.ctx, *args, g2=(e.h, e.tau_h))
    return PlonkKzgSnark.verify_each(e.ctx, *args, g2=(e.h, e.tau_h))


def job(jobs, e, proofs, links, combined):
    return jobs.wait(jobs.submit_verify([p[0] for p in proofs], [p[1] for p in proofs], [p[2] for p in proofs], links,
                                        combined=combined, g2=(e.h, e.tau_h)))


def pool_stats(lib, handle):
    out = (C.c_uint64 * 4)()
    assert lib.b200_pool_stats(handle, out) == OK
    return list(out)


@pytest.mark.parametrize("combined", [False, True])
def test_verdicts_equal_the_bare_context(env, pool, box, combined):
    e = env
    for k, seed in ((1, None), (16, 160), (64, 640)):
        proofs, links = e.orders(k, seed)
        want = bare(e, proofs, links, combined)
        verdicts = want[1] if combined else want
        if seed is None:
            assert all(verdicts) and len(verdicts) == 3 * k
        else:
            assert 0 < verdicts.count(False) < len(verdicts), k
        before = pool.stats()
        assert job(pool, e, proofs, links, combined) == want, (k, combined)
        after = pool.stats()
        assert after["submitted"] == before["submitted"] + 1 and after["completed"] == before["completed"] + 1
        assert after["failed"] == before["failed"]
        t = box.submit_verify([p[0] for p in proofs], [p[1] for p in proofs], [p[2] for p in proofs], links,
                              combined=combined, g2=(e.h, e.tau_h))
        assert box.ticket_device(t) in range(len(box.devices))
        assert box.wait(t) == want, (k, combined)


def test_every_tampering_kind(env, pool):
    e = env
    for kind in KINDS:
        proofs, links = e.orders(4)
        if kind == "link_layout":
            links[2] = tamper_link(links[2])
        else:
            proofs[5] = tamper_proof(proofs[5], kind)
        want = bare(e, proofs, links, False)
        assert want.count(False) == 1, kind
        assert job(pool, e, proofs, links, False) == want, kind
        ok, verdicts = job(pool, e, proofs, links, True)  # one failing item: the bisection runs inside the job
        assert (ok, verdicts) == bare(e, proofs, links, True) and not ok and verdicts == want, kind


def test_all_failing_and_zero_items(env, pool, box):
    e = env
    proofs, links = e.orders(8)
    proofs = [tamper_proof(p, "eval_bit") for p in proofs]
    links = [tamper_link(l_) for l_ in links]
    assert job(pool, e, proofs, links, False) == bare(e, proofs, links, False) == [False] * 24
    assert job(pool, e, proofs, links, True) == bare(e, proofs, links, True) == (False, [False] * 24)
    for jobs in (pool, box):
        assert job(jobs, e, [], [], False) == []
        assert job(jobs, e, [], [], True) == (True, [])
    # the C call with no arrays at all: B200_OK, all_accepted 1
    lib, t, ok = pool._lib, C.c_uint64(), C.c_int(7)
    h, tau_h = (a.ctypes.data_as(C.c_void_p) for a in (e.h, e.tau_h))
    assert lib.b200_pool_submit_verify(pool._h, 1, None, 0, None, 0, None, 0, h, tau_h, C.byref(ok), None, C.byref(t)) == OK
    assert lib.b200_pool_wait(pool._h, t.value) == OK and ok.value == 1


def _overwrite(obj):
    """Every numpy array and ctypes object reachable from obj is filled with 0xFF bytes."""
    if isinstance(obj, np.ndarray):
        obj.view(np.uint8)[...] = 0xFF
    elif isinstance(obj, (C.Structure, C.Array)):
        C.memset(C.addressof(obj), 0xFF, C.sizeof(obj))
    elif isinstance(obj, (tuple, list)):
        for x in obj:
            _overwrite(x)


@pytest.mark.parametrize("mode", [0, 1])
def test_inputs_overwritten_after_submit(env, pool, mode):
    """The raw C call: every input array, struct and G2 record is overwritten as soon as the submit returns, while the
    pool is still busy with proofs queued before the job."""
    e = env
    proofs, links = e.orders(16, seed=1600 + mode)
    want = bare(e, proofs, links, mode == 1)
    proofs = [(vk, np.array(pi, dtype=np.uint64).copy(), B200Proof.from_buffer_copy(bytes(p))) for vk, pi, p in proofs]
    links = [(np.array(a).copy(), np.array(b).copy(), B200LinkProof.from_buffer_copy(bytes(lp)), lay) for a, b, lp, lay in links]
    busy = [pool.submit_prove_witness(e.s.pks[j], e.s.circs[j].witness, e.bl[j]) for j in (1, 2, 3, 4)]
    b = _VerifyBatch([p[0] for p in proofs], [p[1] for p in proofs], [p[2] for p in proofs], links, None)
    verdicts = (C.c_uint8 * b.n_c)()
    ok, t = C.c_int(5), C.c_uint64()
    assert pool._lib.b200_pool_submit_verify(pool._h, mode, *b.args, C.byref(ok) if mode else None, verdicts, C.byref(t)) == OK
    _overwrite(b.keep)
    _overwrite([[p[1], p[2]] for p in proofs] + [[x[0], x[1], x[2]] for x in links])
    del b.keep, b.args
    for tk in busy:
        pool.wait(tk)
    assert pool._lib.b200_pool_wait(pool._h, t.value) == OK
    got = b.verdicts(verdicts)
    assert (got if mode == 0 else (bool(ok.value), got)) == want


def test_interleaved_with_proof_jobs_from_two_threads(env, pool):
    """One thread submits prove, bundle and settlement jobs, another verification jobs, all on the same pool: every proof,
    link proof and public-input vector equals the single calls' on the session context, and every verdict list equals
    the bare-context one."""
    e = env
    s = e.s
    settle_links = [(e.hints[a], lay) for a, b, lay in s.links]
    cases = [(k, seed, combined) for k in (1, 4, 16) for seed in (None, 7 * k) for combined in (False, True)]
    wants = [bare(e, *e.orders(k, seed), combined) for k, seed, combined in cases]
    errors = []

    def provers():
        try:
            for rnd in range(2):
                tk = [pool.submit_prove_witness(pk, c.witness, b) for pk, c, b in zip(s.pks, s.circs, e.bl)]
                tb = pool.submit_bundle_witness(s.bases, [(pk, c.witness, b) for pk, c, b in zip(s.pks, s.circs, e.bl)], s.links)
                ts = pool.submit_settlement_witness(s.bases, s.pks[0], s.circs[0].witness, e.bl[0], settle_links)
                for j, t in enumerate(tk):
                    proof, pub = pool.wait(t)
                    assert bytes(proof) == bytes(e.proofs[j]) and pub.tobytes() == e.pubs[j].tobytes(), (rnd, j)
                proofs, _, lps, _ = pool.wait(tb)
                assert [bytes(p) for p in proofs] == [bytes(p) for p in e.proofs], rnd
                assert [bytes(x) for x in lps] == [bytes(x) for x in e.link_proofs], rnd
                proof, lps, st, _ = pool.wait(ts)
                assert st == [OK] * (len(lps) + 1) and bytes(proof) == bytes(e.proofs[0]), rnd
                assert [bytes(x) for x in lps] == [bytes(x) for x in e.link_proofs], rnd
        except Exception as exc:  # noqa: BLE001  (reported by the main thread)
            errors.append(exc)

    def verifiers():
        try:
            for rnd in range(2):
                tickets = []
                for k, seed, combined in cases:
                    proofs, links = e.orders(k, seed)
                    tickets.append(pool.submit_verify([p[0] for p in proofs], [p[1] for p in proofs], [p[2] for p in proofs],
                                                      links, combined=combined, g2=(e.h, e.tau_h)))
                for t, want, case in zip(tickets, wants, cases):
                    assert pool.wait(t) == want, (rnd, case)
        except Exception as exc:  # noqa: BLE001
            errors.append(exc)

    threads = [threading.Thread(target=provers), threading.Thread(target=verifiers)]
    for th in threads:
        th.start()
    for th in threads:
        th.join()
    assert not errors, errors
    assert pool._lib.b200_pool_wait_all(pool._h) == OK


def test_refusals_at_submit_queue_nothing(env, pool, box):
    e = env
    lib = pool._lib
    proofs, links = e.orders(2)
    b = _VerifyBatch([p[0] for p in proofs], [p[1] for p in proofs], [p[2] for p in proofs], links, None)
    vks, n_vks, c_proofs, n_proofs, c_links, n_links, h, tau_h = b.args
    verdicts, ok, t = (C.c_uint8 * b.n_c)(), C.c_int(), C.c_uint64(99)
    box_pools = [lib.b200_box_pool(box._h, i) for i in range(len(box.devices))]

    def refused(code, msg, *args, fn=None, handle=None):
        fn = fn or lib.b200_pool_submit_verify
        handle = pool._h if handle is None else handle
        before = [pool_stats(lib, pool._h)] + [pool_stats(lib, p) for p in box_pools]
        assert fn(handle, *args) == code, msg
        assert msg in lib.b200_last_error(), (msg, lib.b200_last_error())
        assert [pool_stats(lib, pool._h)] + [pool_stats(lib, p) for p in box_pools] == before, msg

    def call(mode=0, v=vks, nv=n_vks, p=c_proofs, np_=n_proofs, l_=c_links, nl=n_links, g2h=h, g2t=tau_h, out=verdicts,
             tk=C.byref(t)):
        return (mode, v, nv, p, np_, l_, nl, g2h, g2t, C.byref(ok), out, tk)

    assert lib.b200_pool_submit_verify(None, *call()) == INVALID and b"null pool" in lib.b200_last_error()
    assert lib.b200_box_submit_verify(None, *call()) == INVALID and b"null box" in lib.b200_last_error()
    refused(INVALID, b"null ticket", *call(tk=None))
    refused(INVALID, b"mode must be 0 or 1", *call(mode=2))
    refused(INVALID, b"null vks", *call(v=None))
    refused(INVALID, b"null proofs", *call(p=None))
    refused(INVALID, b"null links", *call(l_=None))
    refused(INVALID, b"null verdicts", *call(out=None))
    refused(INVALID, b"null G2 record", *call(g2h=None))
    # item checks, each naming the entry
    one = lambda arr, i, **kw: (type(arr[0]) * len(arr))(*[type(arr[0])(**{**{f: getattr(x, f) for f, _ in x._fields_},  # noqa: E731
                                                                            **(kw if j == i else {})})
                                                         for j, x in enumerate(arr)])
    refused(INVALID, b"bad proof entry 3", *call(p=one(c_proofs, 3, vk=n_vks)))
    refused(INVALID, b"bad proof entry 1", *call(p=one(c_proofs, 1, proof=None)))
    refused(INVALID, b"bad verifying key 1", *call(v=one(vks, 1, log_n=29)))
    refused(INVALID, b"bad link entry 1", *call(l_=one(c_links, 1, alignment=29)))
    refused(INVALID, b"bad link entry 0", *call(l_=one(c_links, 0, size=0)))
    refused(INVALID, b"bad link entry 1", *call(l_=one(c_links, 1, comm2=None)))
    # G2 records off the twist: one bit flipped, and a coordinate >= q
    off = np.array(e.h, dtype=np.uint64).copy()
    off[0] ^= np.uint64(1)
    big = np.array(e.tau_h, dtype=np.uint64).copy()
    big[4:8] = vm.to_words(vm.to_int(big[4:8]) + vm.Q)
    for bad, where in ((off, "g2h"), (big, "g2t")):
        refused(NOT_ON_CURVE, b"G2 point not on curve", *call(**{where: bad.ctypes.data_as(C.c_void_p)}))
        refused(NOT_ON_CURVE, b"G2 point not on curve", *call(**{where: bad.ctypes.data_as(C.c_void_p)}),
                fn=lib.b200_box_submit_verify, handle=box._h)
    refused(INVALID, b"mode must be 0 or 1", *call(mode=-1), fn=lib.b200_box_submit_verify, handle=box._h)
    assert t.value == 99 and not any(verdicts)


def test_singleprover_batch_on_a_pool_and_a_box(ctx, pool, box, srs_2_16, srs_2_16_g2):
    """`circuit_types.batch_verify_singleprover_proofs` with `pool=` / `box=`: the combined check as one job, failing
    indices named as on the system context."""
    import renegade_b200 as rb
    from host_circuits import statements as st
    from host_circuits import valid_balance_create as vbc
    from renegade_b200 import circuit_types as ct
    params = rb.parse_ptau_file(ctx, srs_2_16, count=(1 << 14) + 3)
    ct.set_system_srs(ctx, params.powers_of_g, *srs_2_16_g2)
    try:
        items = []
        for seed in (7, 8):
            w, s = vbc.create_witness_statement(seed)
            items.append((st.ValidBalanceCreate, s, ct.singleprover_prove(st.ValidBalanceCreate, w, s)))
        wrong = [items[0], (items[1][0], items[0][1], items[1][2])]  # proof 1 under statement 0
        for jobs in ({"pool": pool}, {"box": box}):
            ct.batch_verify_singleprover_proofs(items, **jobs)
            with pytest.raises(ct.VerifierError) as err:
                ct.batch_verify_singleprover_proofs(wrong, **jobs)
            assert "[1]" in str(err.value), jobs
        with pytest.raises(ValueError):
            ct.batch_verify_singleprover_proofs(items, pool=pool, box=box)
    finally:
        ct.clear_key_cache()
