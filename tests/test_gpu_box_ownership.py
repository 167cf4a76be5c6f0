"""GPU: a box refuses proving keys and SRS tables that another box made.  A key of a box over as many devices, and an SRS
of a box over fewer or as many devices, are B200_ERR_INVALID at submit for every box entry that takes one, and a refusal
queues nothing on any pool.  Such a key or SRS holds memory of the other box's contexts, and an SRS of a smaller box has
no table for some of this box's devices.  The box's own keys and SRS still make the single-context proofs."""
import ctypes as C

import numpy as np
import pytest

from renegade_b200 import _lib, synth
from renegade_b200.backend import (BundleProof, GroupLayout, LinkingHint, PlonkKzgSnark, ProverBox, ProverError,
                                   link_proofs)
from test_gpu_verify_jobs import pool_stats

pytestmark = pytest.mark.gpu
INVALID = _lib.B200_ERR_INVALID
TAU = 0x0c1d2e3f405162738495a6b7c8d9eafb0c1d2e3f405162738495a6b7c8d9eafb
LOG_N = 10
LAYOUT = GroupLayout(alignment=7, offset=20, size=9)


@pytest.fixture(scope="module")
def env(oracle, pyoracle):
    """Two 2^10 circuits sharing a link group, their SRS, and three boxes of one worker per device: `one` over [0], `two`
    over [0, 0] and `other` over [0], each with its SRS."""
    vals = [(i * 0xD1B54A32D192ED03 + 99) % synth.R for i in range(LAYOUT.size)]
    circs = [synth.synth_circuit(LOG_N, num_inputs=6, seed=31 + i, link=(LAYOUT.alignment, LAYOUT.offset, vals))
             for i in range(2)]
    tau = oracle.int_to_limbs(pyoracle.to_mont(TAU % pyoracle.R, pyoracle.R))
    points = oracle.srs_from_tau(tau, (1 << LOG_N) + 3)
    boxes = {name: ProverBox(devices, workers_per_device=1) for name, devices in (("one", [0]), ("two", [0, 0]),
                                                                                   ("other", [0]))}
    srs = {name: box.load_srs(points) for name, box in boxes.items()}
    try:
        yield circs, points, boxes, srs
    finally:
        for name, box in boxes.items():
            box.free_srs(srs[name])
            box.close()


def all_stats(boxes):
    lib = _lib.load()
    return [pool_stats(lib, lib.b200_box_pool(b._h, i)) for b in boxes.values() for i in range(len(b.devices))]


def refused(boxes, fn, *args):
    """fn(*args) raises B200Error INVALID naming another box, and no pool of any box got a job"""
    before = all_stats(boxes)
    with pytest.raises(ProverError) as err:
        fn(*args)
    assert err.value.code == INVALID and "another box" in str(err.value), str(err.value)
    assert all_stats(boxes) == before


def key(box, srs, c):
    return box.preprocess(srs, c.log_n, c.num_inputs, c.selectors, c.perm, c.k)


def test_a_key_of_another_box_with_as_many_devices_is_refused(env):
    circs, _, boxes, srs = env
    one, other, lib = boxes["one"], boxes["other"], _lib.load()
    c = circs[0]
    own, stranger = key(one, srs["one"], c), key(other, srs["other"], c)
    try:
        wires = np.ascontiguousarray(c.wires, dtype=np.uint64)
        pub = np.ascontiguousarray(c.pub_inputs, dtype=np.uint64)
        bl = synth.splitmix_blinders(5)
        proof = _lib.STRUCTS["b200_proof"]()
        ptr = lambda a: a.ctypes.data_as(C.c_void_p)  # noqa: E731
        t = C.c_uint64(7)

        def prove(pk):
            _lib.check(lib.b200_box_submit_prove(one._h, pk, ptr(wires), ptr(pub), c.num_inputs, ptr(bl), C.byref(proof),
                                                 None, C.byref(t)))

        def bundle(*pks):
            arr = (BundleProof * len(pks))(*[BundleProof(None, ptr(wires), ptr(pub), c.num_inputs, ptr(bl),
                                                         C.cast(C.pointer(proof), C.c_void_p), None) for _ in pks])
            _lib.check(lib.b200_box_submit_bundle(one._h, srs["one"], (C.c_void_p * len(pks))(*pks), arr, len(pks), None, 0,
                                                  C.byref(t)))

        refused(boxes, prove, stranger)
        refused(boxes, bundle, stranger)
        refused(boxes, bundle, own, stranger)
        assert t.value == 7
        with pytest.raises(ProverError, match="not made by this box"):  # the wrapper refuses it before the library
            one.submit_prove(stranger, wires.ctypes.data, c.pub_inputs, bl)
    finally:
        one.free_pk(own)
        other.free_pk(stranger)


def test_an_srs_of_another_box_is_refused(env):
    """The SRS of `one` (one device) on `two` (two devices) for every entry that takes an SRS, and the SRS of a box with
    as many devices, or more, on a bundle."""
    circs, _, boxes, srs = env
    two, one = boxes["two"], boxes["one"]
    c = circs[0]
    pk = key(two, srs["two"], c)
    wpk = two.preprocess_wiring(srs["two"], c.log_n, c.num_inputs, c.selectors, c.wire_vars, c.num_vars, c.k)
    own = key(one, srs["one"], c)
    try:
        wires = np.ascontiguousarray(c.wires, dtype=np.uint64)
        bl = synth.splitmix_blinders(6)
        hint = LinkingHint(np.zeros(((1 << LOG_N) + 2, 4), dtype=np.uint64), np.zeros(8, dtype=np.uint64))
        entry = (pk, wires.ctypes.data, c.pub_inputs, bl)
        small = srs["one"]
        refused(boxes, two.submit_bundle, small, [entry, entry], [(0, 1, LAYOUT)])
        refused(boxes, two.submit_bundle, small, [entry], [])
        refused(boxes, two.preprocess, small, c.log_n, c.num_inputs, c.selectors, c.perm, c.k)
        refused(boxes, two.preprocess_wiring, small, c.log_n, c.num_inputs, c.selectors, c.wire_vars, c.num_vars, c.k)
        refused(boxes, two.submit_settlement, small, pk, wires, c.pub_inputs, bl, [(hint, LAYOUT)])
        refused(boxes, two.submit_settlement_witness, small, wpk, c.witness, bl, [(hint, LAYOUT)])
        for stranger in (srs["two"], srs["other"]):
            refused(boxes, one.submit_bundle, stranger, [(own, wires.ctypes.data, c.pub_inputs, bl)], [])
    finally:
        two.free_pk(pk)
        two.free_pk(wpk)
        one.free_pk(own)


def test_own_keys_still_make_single_context_proofs(ctx, env):
    circs, points, boxes, srs = env
    two = boxes["two"]
    bases = ctx.load_bases(points)
    spks = [PlonkKzgSnark.preprocess(ctx, bases, LOG_N, c.num_inputs, c.selectors, c.perm, c.k) for c in circs]
    pks = [key(two, srs["two"], c) for c in circs]
    try:
        wires = [np.ascontiguousarray(c.wires, dtype=np.uint64) for c in circs]
        bl = [synth.splitmix_blinders(80 + i) for i in range(4)]
        singles = [PlonkKzgSnark.prove_with_link_hint(ctx, spks[i % 2], circs[i % 2].wires, circs[i % 2].pub_inputs, b)
                   for i, b in enumerate(bl)]
        tickets = [two.submit_prove(pks[i % 2], wires[i % 2].ctypes.data, circs[i % 2].pub_inputs, b,
                                    with_link_poly=(i < 2), keep=wires[i % 2]) for i, b in enumerate(bl)]
        assert {two.ticket_device(t) for t in tickets} == {0, 1}
        for i, t in enumerate(tickets):
            got = two.wait(t)
            proof, hint = singles[i]
            if i < 2:
                got, poly = got
                assert (poly == hint.linking_wire_poly).all()
            assert bytes(got) == bytes(proof), i
        t = two.submit_bundle(srs["two"], [(pks[i], wires[i].ctypes.data, circs[i].pub_inputs, bl[i]) for i in (0, 1)],
                              [(0, 1, LAYOUT)])
        proofs, polys, links = two.wait(t)
        for i in (0, 1):
            assert bytes(proofs[i]) == bytes(singles[i][0]) and (polys[i] == singles[i][1].linking_wire_poly).all()
        direct, _ = link_proofs(ctx, bases, singles[0][1], singles[1][1], LAYOUT)
        assert bytes(links[0]) == bytes(direct)
    finally:
        for pk in pks:
            two.free_pk(pk)
        for spk in spks:
            spk.free()
