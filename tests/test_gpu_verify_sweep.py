"""The device verifiers over the sweep of `verify_sweep.py`: every domain 2^2 ... 2^17 (0, 1, 5 and all public inputs),
every link layout of `link_layouts.py`, and each item's tampered twins, in one call, with keys of sixteen sizes mixed and
honest and tampered items sharing warps in every order.  `verify_each` on both sides of the switch from the 16-lane
pairing to the one-thread kernel, `batch_verify`'s verdicts, and a pool's and a box's verification job give every item
the verdict the single host verifier and the oracle give it (`test_verify_sweep_cpu.py`).  The oracle's own pairing
operands (A, -B) of every proof item through `pairing_check_many` separate the device pairing from the device's G1
side.  And the C entry points refuse a link group of more roots than its subgroup holds, with nothing queued or
written."""
import ctypes as C

import numpy as np
import pytest

import verify_sweep as vs
from renegade_b200 import _lib
from renegade_b200.backend import (B200LinkProof, B200Proof, GroupLayout, PlonkKzgSnark, ProverBox, ProverPool,
                                   VerifyingKey, _VerifyBatch, pairing_check_many)
from test_gpu_pairing_warp import wave
from test_gpu_verify_jobs import pool_stats

pytestmark = pytest.mark.gpu
Q = 0x30644E72E131A029B85045B68181585D97816A916871CA8D3C208C16D87CFD47


@pytest.fixture(scope="module")
def sweep(oracle):
    return vs.build(oracle)


def call_args(sw, proofs, links):
    """(vks, pub_inputs, proofs, links) of the verifier calls, and the expected verdicts, proofs first"""
    vks = [VerifyingKey(*vs.vk_parts(sw, it), sw.h, sw.tau_h) for it in proofs]
    args = (vks, [it.pi for it in proofs], [B200Proof.from_buffer_copy(it.proof.tobytes()) for it in proofs],
            [(it.c1, it.c2, B200LinkProof.from_buffer_copy(it.lp.tobytes()), GroupLayout(*it.layout)) for it in links])
    return args, [it.want for it in proofs] + [it.want for it in links]


def names(sw, proofs, links, got, want):
    items = list(proofs) + list(links)
    return [items[i].name for i in range(len(want)) if got[i] != want[i]][:8]


def tiled(items, n):
    return [items[i % len(items)] for i in range(n)]


def test_verify_each_below_the_switch(ctx, sweep):
    sw = sweep
    args, want = call_args(sw, sw.proofs, sw.links)
    assert len(want) <= wave() and len(sw.proofs) % 2 == 0  # the links' pairs start on an even item too
    assert {"HT", "TH", "HH"} <= set(vs.pair_kinds(want))
    got = PlonkKzgSnark.verify_each(ctx, *args, g2=(sw.h, sw.tau_h))
    assert got == want, names(sw, sw.proofs, sw.links, got, want)


def test_verify_each_above_the_switch(ctx, sweep):
    sw = sweep
    k = wave() + 1
    n_links = k // 4
    proofs, links = tiled(sw.proofs, k - n_links), tiled(sw.links, n_links)
    args, want = call_args(sw, proofs, links)
    got = PlonkKzgSnark.verify_each(ctx, *args, g2=(sw.h, sw.tau_h))
    assert got == want, names(sw, proofs, links, got, want)


def test_batch_verify_verdicts(ctx, sweep):
    sw = sweep
    args, want = call_args(sw, sw.proofs, sw.links)
    ok, got = PlonkKzgSnark.batch_verify(ctx, *args, g2=(sw.h, sw.tau_h))
    assert not ok and got == want, names(sw, sw.proofs, sw.links, got, want)
    honest = [it for it in sw.proofs if it.want], [it for it in sw.links if it.want]
    args, want = call_args(sw, *honest)
    assert PlonkKzgSnark.batch_verify(ctx, *args, g2=(sw.h, sw.tau_h)) == (True, want) and all(want)


def test_pool_and_box_verification_jobs(sweep):
    sw = sweep
    args, want = call_args(sw, sw.proofs, sw.links)
    pool = ProverPool(0, workers=2)
    try:
        assert pool.wait(pool.submit_verify(*args, g2=(sw.h, sw.tau_h))) == want
    finally:
        pool.close()
    box = ProverBox([0], workers_per_device=2)
    try:
        assert box.wait(box.submit_verify(*args, g2=(sw.h, sw.tau_h))) == want
    finally:
        box.close()


def _neg(xy):
    out = np.array(xy, dtype=np.uint64).copy()
    if out.any():
        y = int.from_bytes(out[4:8].tobytes(), "little")
        out[4:8] = np.frombuffer(((Q - y) % Q).to_bytes(32, "little"), dtype=np.uint64)
    return out


@pytest.mark.parametrize("where", ["below", "above"])
def test_oracle_operands_through_the_device_pairing(ctx, sweep, oracle, where):
    """e(A, tau H) e(-B, H) == 1 for the oracle's A and B of every proof item: the oracle's known-tau verdict"""
    sw = sweep
    g1, want = [], []
    for it in sw.proofs:
        lg, ni, k, _, _ = vs.vk_parts(sw, it)
        pk = sw.keys[it.key].pk
        proof = oracle.PlonkProof.from_buffer_copy(it.proof.tobytes())
        (a, a_inf), (b, b_inf) = oracle.plonk_verify_operands(lg, ni, k, pk, it.pi, proof)
        zero = np.zeros(8, dtype=np.uint64)
        g1.append([zero if a_inf else a, zero if b_inf else _neg(b)])
        want.append(oracle.plonk_verify_known_tau(lg, ni, k, pk, it.pi, proof, sw.tau))
    assert want == [it.want for it in sw.proofs]
    g1, want = np.array(g1, dtype=np.uint64), np.array(want)
    n = len(want) if where == "below" else wave() + 1
    idx = np.arange(n) % len(want)
    got = pairing_check_many(ctx, np.stack([sw.tau_h, sw.h]), g1[idx])
    assert (got == want[idx]).all(), [sw.proofs[i % len(want)].name for i in np.nonzero(got != want[idx])[0][:8]]


def test_c_entry_points_refuse_a_group_larger_than_its_subgroup(ctx, sweep):
    """link 1 at alignment 3 with 9 roots: every entry point refuses it and names it, writes no verdict and queues no
    job (9 products even where it was not refused: safe to run)"""
    sw = sweep
    proofs = sw.proofs[:2]
    args, want = call_args(sw, proofs, sw.links[:2])
    b = _VerifyBatch(*args, (sw.h, sw.tau_h), "verify_each")
    b.args[4][1].alignment, b.args[4][1].size = 3, 9
    lib = ctx._lib
    sentinel = [0x5A] * b.n_c
    verdicts, ok = (C.c_uint8 * b.n_c)(*sentinel), C.c_int(7)
    assert lib.b200_plonk_verify_each(ctx._h, *b.args, verdicts) == _lib.B200_ERR_INVALID
    assert b"verify_each: bad link entry 1" in lib.b200_last_error() and list(verdicts) == sentinel
    assert lib.b200_plonk_batch_verify(ctx._h, *b.args, C.byref(ok), verdicts) == _lib.B200_ERR_INVALID
    assert b"batch_verify: bad link entry 1" in lib.b200_last_error() and list(verdicts) == sentinel and ok.value == 0
    pool, box = ProverPool(0, workers=1), ProverBox([0], workers_per_device=1)
    try:
        handles = [pool._h, lib.b200_box_pool(box._h, 0)]
        for fn, h in ((lib.b200_pool_submit_verify, pool._h), (lib.b200_box_submit_verify, box._h)):
            for mode in (0, 1):
                before = [pool_stats(lib, x) for x in handles]
                t = C.c_uint64(99)
                assert fn(h, mode, *b.args, C.byref(ok), verdicts, C.byref(t)) == _lib.B200_ERR_INVALID
                assert b"bad link entry 1" in lib.b200_last_error()
                assert [pool_stats(lib, x) for x in handles] == before and t.value == 99 and list(verdicts) == sentinel
    finally:
        pool.close()
        box.close()
    # the context still verifies
    assert PlonkKzgSnark.verify_each(ctx, *args, g2=(sw.h, sw.tau_h)) == want
