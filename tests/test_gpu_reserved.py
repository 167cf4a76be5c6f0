"""Reserved SMs for the express lane (include/b200reserved.h): a pool whose express workers run on a green-context group
of SMs of their own and whose normal workers run on the rest.  Placement is checked with `probe_sms` masks (which SMs a
kernel's blocks reached, eagerly and under graph replay), not with timings; every job kind gives the bare context's bytes
on either group, expedited or not; keys and SRS tables made on one group serve the other."""
import ctypes as C

import pytest
import torch

from renegade_b200 import _lib, synth
from renegade_b200.backend import PlonkKzgSnark, ProverBox, ProverPool
from test_gpu_express import Env, as_bytes, kinds
from test_gpu_prove_witness import TAU, load_srs

pytestmark = pytest.mark.gpu
INVALID = _lib.B200_ERR_INVALID
EXPRESS = 1  # worker index of the first express worker of a pool with one normal worker


@pytest.fixture(scope="module")
def env(ctx, oracle, pyoracle, srs_2_16_g2):
    e = Env(ctx, oracle, pyoracle, srs_2_16_g2)
    yield e
    e.free()


def device_sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def test_a_key_made_on_the_normal_group_proves_on_the_express_group(env, ctx, oracle, pyoracle):
    """Memory is the device's: a key and an SRS made on a normal worker's context prove on the express worker (and on the
    normal one), with the bare context's bytes."""
    c = synth.synth_circuit(10, num_inputs=2, seed=7701)
    pool = ProverPool(0, workers=1, express=1, express_sms=16)
    try:
        pctx = pool.context(0)
        bases, bare_bases = load_srs(pctx, oracle, pyoracle, c.n), load_srs(ctx, oracle, pyoracle, c.n)
        pk = PlonkKzgSnark.preprocess_wiring(pctx, bases, c.log_n, c.num_inputs, c.selectors, c.wire_vars, c.num_vars, c.k)
        bare_pk = PlonkKzgSnark.preprocess_wiring(ctx, bare_bases, c.log_n, c.num_inputs, c.selectors, c.wire_vars, c.num_vars,
                                                  c.k)
        bl = synth.splitmix_blinders(7702)
        want = as_bytes(PlonkKzgSnark.prove_witness(ctx, bare_pk, c.witness, bl)[0])
        for w in (0, EXPRESS):
            blocker = env.block(pool) if w == EXPRESS else None
            t = pool.submit_prove_witness(pk, c.witness, bl)
            if w == EXPRESS:
                assert pool.expedite(t) == 1
            got, _, worker = pool.wait_info(t)
            assert worker == w and as_bytes(got[0]) == want, w
            if blocker:
                pool.wait(blocker)
        pk.free()
        bare_pk.free()
        bases.free()
        bare_bases.free()
    finally:
        pool.close()


@pytest.mark.parametrize("express_sms", [8, 16, 24])
def test_partition_and_placement(env, express_sms):
    pool = ProverPool(0, workers=2, express=2, express_sms=express_sms)
    try:
        normal, express = pool.partition()
        # the express group is a split group (multiples of 8); the normal group is every SM left, 124 of an H100 SXM's 132
        assert express >= express_sms and express % 8 == 0 and normal >= 8, (normal, express)
        assert normal + express <= device_sms() and normal >= device_sms() - express - 7
        c0 = env.s.circs[0]
        for rnd in range(2):  # before any proof (main and companion streams), then after proofs (side stream, graphs)
            n_set = pool.probe_sms(0) | pool.probe_sms(1)
            e_set = pool.probe_sms(2) | pool.probe_sms(3)
            assert n_set and e_set and not n_set & e_set, rnd
            assert len(n_set) <= normal and len(e_set) <= express, (rnd, len(n_set), len(e_set))
            assert max(n_set | e_set) < device_sms()
            for i in range(3):  # eager, captured, replayed on every worker
                ts = [pool.submit_prove_witness(env.s.pks[0], c0.witness, env.bl[0]) for _ in range(2)]
                ts += [pool.submit_prove_witness(env.s.pks[0], c0.witness, env.bl[0]) for _ in range(2)]
                for t in ts[2:]:
                    pool.expedite(t)
                for t in ts:
                    pool.wait(t)
    finally:
        pool.close()
    assert ProverPool(0, workers=1, express=1).partition() == (0, 0)


def test_every_job_kind_on_both_groups(env):
    lib = _lib.load()
    pool = ProverPool(0, workers=1, express=1, express_sms=16)
    try:
        for name, submit, bare, n_jobs in kinds(env):
            want = as_bytes(bare())
            t = submit(pool)  # not expedited: the normal worker on the normal group
            got, _, worker = pool.wait_info(t)
            assert worker == 0 and as_bytes(got) == want, name
            blocker = env.block(pool)
            t = submit(pool)
            assert pool.expedite(t) == n_jobs, name
            got, done_at, worker = pool.wait_info(t)
            _, blocker_done_at, _ = pool.wait_info(blocker)
            assert worker == EXPRESS and done_at < blocker_done_at, name
            assert as_bytes(got) == want, name
        # a warm proof on the express worker replays its captured rounds: 7 graph submissions
        c0 = env.s.circs[0]
        want = as_bytes(PlonkKzgSnark.prove_witness(env.ctx, env.s.pks[0], c0.witness, env.bl[2])[:1])
        for i in range(3):
            blocker = env.block(pool)
            g0 = lib.b200_graph_launches()
            t = pool.submit_prove_witness(env.s.pks[0], c0.witness, env.bl[2])
            assert pool.expedite(t) == 1
            got, _, worker = pool.wait_info(t)
            g1 = lib.b200_graph_launches()
            assert worker == EXPRESS and as_bytes(got[:1]) == want, i
            pool.wait(blocker)
        assert g1 - g0 == 7
    finally:
        pool.close()


def test_box_gives_the_pool_bytes(env, oracle, pyoracle):
    c0 = env.s.circs[0]
    box = ProverBox([0], workers_per_device=1, express_per_device=1, express_sms=16)
    try:
        tau = oracle.int_to_limbs(pyoracle.to_mont(TAU % pyoracle.R, pyoracle.R))
        srs = box.load_srs(oracle.srs_from_tau(tau, c0.n + 3))
        pk = box.preprocess_wiring(srs, c0.log_n, c0.num_inputs, c0.selectors, c0.wire_vars, c0.num_vars, c0.k)
        want = PlonkKzgSnark.prove_witness(env.ctx, env.s.pks[0], c0.witness, env.bl[1])
        want = as_bytes((want[0], want[1].linking_wire_poly, want[2]))
        for expedite in (False, True):
            t = box.submit_prove_witness(pk, c0.witness, env.bl[1], with_link_poly=True)
            if expedite:
                box.expedite(t)
            (proof, poly, pub), _, _ = box.wait_info(t)
            assert as_bytes((proof, poly, pub)) == want, expedite
        box.free_pk(pk)
        box.free_srs(srs)
    finally:
        box.close()


def test_refusals_and_lifecycle(env):
    lib = _lib.load()
    h = C.c_void_p()
    sms = device_sms()
    too_many = (sms - 4) // 8 * 8 + 8  # rounds past the device: fewer than 8 SMs left
    for n, x, r in ((1, 1, 0), (1, 1, 12), (1, 0, 16), (0, 1, 16), (1, 1, 256), (1, 1, too_many), (1, 1, sms // 8 * 8)):
        assert lib.b200_pool_create_reserved(0, n, x, r, C.byref(h)) == INVALID and not h.value, (n, x, r)
    assert b"8 SMs" in lib.b200_last_error()
    devs = (C.c_int * 1)(0)
    assert lib.b200_box_create_reserved(devs, 1, 1, 1, 4, C.byref(h)) == INVALID and not h.value
    c0 = env.s.circs[0]
    want = as_bytes(PlonkKzgSnark.prove_witness(env.ctx, env.s.pks[0], c0.witness, env.bl[0])[:1])
    for _ in range(3):
        pool = ProverPool(0, workers=2, express=1, express_sms=8)
        t = pool.submit_prove_witness(env.s.pks[0], c0.witness, env.bl[0])
        pool.wait(t)
        pool.close()
    pool = ProverPool(0, workers=2, express=1, express_sms=8)
    try:
        for expedite in (False, True, True):
            t = pool.submit_prove_witness(env.s.pks[0], c0.witness, env.bl[0])
            if expedite:
                pool.expedite(t)
            assert as_bytes(pool.wait(t)[:1]) == want
    finally:
        pool.close()
