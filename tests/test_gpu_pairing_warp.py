"""The latency path of the device pairing checks (`k_pairing_warp`, `renegade_b200/csrc/pairing_warp.cuh`): each check's
Fq12 arithmetic spread over 16 lanes while the checks fit in one wave of the device, the one-thread kernel past that.
`b200_selftest_pairing` finds no operation that differs from the one-thread functions; `pairing_check_many` equals the
host `b200_pairing_check` check by check on both sides of the switch, at every pair count, with identity points in
any slot, on bilinear triples and their one-point twins, and refuses off-curve points as documented; `verify_each`
equals the single verifiers item by item on both sides of the switch for every tampering kind of
`verify_mutations.py`; and a pool's verification job gives the same verdicts."""
import os
import re

import numpy as np
import pytest
import torch

import pairing_cases as pc
import renegade_b200 as rb
import verify_mutations as vm
from renegade_b200 import _lib, synth
from renegade_b200.backend import (B200LinkProof, B200Proof, GroupLayout, PlonkKzgSnark, ProverPool, VerifyingKey,
                                   link_proofs, pairing_check, pairing_check_many, verify_link_proof)

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
Q = pc.Q
R = pc.R
IDENTITY = np.zeros(8, dtype=np.uint64)


def wave() -> int:
    """The largest check count pairing_many_enqueue sends to the group kernel: kPairWarpBlocksPerSm blocks of
    kPairWarpThreads / 16 checks on every SM of the device (verify_batch.cu)."""
    src = open(os.path.join(ROOT, "renegade_b200", "csrc", "verify_batch.cu")).read()
    threads = int(re.search(r"constexpr int kPairWarpThreads = (\d+);", src).group(1))
    blocks = int(re.search(r"constexpr int kPairWarpBlocksPerSm = (\d+);", src).group(1))
    return torch.cuda.get_device_properties(0).multi_processor_count * blocks * threads // 16


def _neg(rec):
    y = int.from_bytes(np.asarray(rec[4:8], dtype="<u8").tobytes(), "little")
    out = np.array(rec, dtype=np.uint64).copy()
    out[4:8] = np.frombuffer(((Q - y) % Q).to_bytes(32, "little"), dtype="<u8")
    return out


def host(g1, g2):
    return np.array([pairing_check(list(c), list(g2)) if len(g2) else True for c in g1], dtype=bool)


def tiled_check(ctx, g2, distinct, n):
    """pairing_check_many over n checks cycling through `distinct` (c, m, 8), against the host answer of each"""
    want = host(distinct, g2)
    idx = np.arange(n) % len(distinct)
    got = pairing_check_many(ctx, g2, distinct[idx])
    assert got.shape == (n,) and (got == want[idx]).all(), [int(i) for i in np.nonzero(got != want[idx])[0][:8]]
    return want


@pytest.fixture(scope="module")
def pts(ctx, srs_head):
    return rb.parse_ptau_file(ctx, srs_head, count=64).powers_of_g_host


@pytest.fixture(scope="module")
def ratio(pts):
    """e(tau^i G, tau H) e(-tau^(i+s) G, H) for i < 40: holds for s = 1 only; s = 2 changes one point"""
    return np.stack([np.stack([pts[i], _neg(pts[i + (1 if i % 3 else 2)])]) for i in range(40)])


@pytest.mark.parametrize("seed", [1, 0xB200, 0x5EED5EED])
def test_selftest_finds_no_mismatch(ctx, seed):
    assert ctx.selftest_pairing(seed, 10_000) == 0


def test_selftest_arguments(ctx):
    import ctypes as C
    lib = _lib.load()
    assert ctx.selftest_pairing(3, 0) == 0
    assert lib.b200_selftest_pairing(None, 1, 1, C.byref(C.c_uint64())) == _lib.B200_ERR_INVALID
    assert lib.b200_selftest_pairing(ctx._h, 1, 1, None) == _lib.B200_ERR_INVALID


@pytest.mark.parametrize("n", [1, 2, 3, 15, 16, 17, 31, 32, 33])
def test_small_counts_equal_the_host(ctx, g2_raw, ratio, n):
    h, tau_h = g2_raw
    want = tiled_check(ctx, np.stack([tau_h, h]), ratio, n)
    assert want.any() and not want.all()


@pytest.mark.parametrize("delta", [-1, 0, 1])
def test_both_sides_of_the_switch(ctx, g2_raw, ratio, delta):
    h, tau_h = g2_raw
    tiled_check(ctx, np.stack([tau_h, h]), ratio, wave() + delta)


def test_every_pair_count_with_identities_anywhere(ctx, g2_raw, ratio):
    h, tau_h = g2_raw
    for m in range(0, 9):
        g2 = np.stack([tau_h, h] * (m // 2) + [h] * (m % 2)) if m else np.zeros((0, 16), dtype=np.uint64)
        rows = []
        for c in range(12):
            row = [ratio[(c + j) % len(ratio)] for j in range(m // 2)]
            row = [p for pair in row for p in pair] + [IDENTITY] * (m % 2)
            if m and c % 4 == 1:
                row[c % m] = IDENTITY  # the identity in a slot that mattered
            if m and c % 4 == 2:
                row = [IDENTITY] * m
            rows.append(row)
        g1 = np.array(rows, dtype=np.uint64).reshape(12, m, 8)
        want = tiled_check(ctx, g2, g1, 12)
        if m == 0:
            assert want.all()


def test_bilinear_triples_and_their_twins(ctx, g2_raw, pts):
    h, tau_h = g2_raw
    P = pc.Points(h)
    a_s, b_s = [3, 5, R - 1, 0xC0FFEE, 2**200 + 7], [2, 7, 11, R - 2, 2**150 + 3]
    for a, b in zip(a_s, b_s):
        g2 = np.stack([P.g2(b), h])
        good = np.stack([P.g1(a), P.g1(-a * b)])
        twin = np.stack([P.g1(a + 1), P.g1(-a * b)])  # one point changed
        got = pairing_check_many(ctx, g2, np.stack([good, twin]))
        assert list(got) == [True, False] and list(got) == list(host(np.stack([good, twin]), g2))
    # the SRS pair in both orders: e(tau^i G, tau H) e(-tau^(i+1) G, H) and e(-tau^(i+1) G, H) e(tau^i G, tau H)
    fwd = np.stack([np.stack([pts[i], _neg(pts[i + 1])]) for i in range(8)])
    rev = fwd[:, ::-1].copy()
    assert pairing_check_many(ctx, np.stack([tau_h, h]), fwd).all()
    assert pairing_check_many(ctx, np.stack([h, tau_h]), rev).all()
    fwd_twin, rev_twin = fwd.copy(), rev.copy()
    fwd_twin[3, 1] = _neg(pts[5])
    rev_twin[6, 0] = _neg(pts[9])
    assert list(pairing_check_many(ctx, np.stack([tau_h, h]), fwd_twin)) == [i != 3 for i in range(8)]
    assert list(pairing_check_many(ctx, np.stack([h, tau_h]), rev_twin)) == [i != 6 for i in range(8)]


def test_off_curve_points_are_refused(ctx, g2_raw, ratio):
    h, tau_h = g2_raw
    g2 = np.stack([tau_h, h])
    for n, c, slot in ((1, 0, 0), (5, 4, 1), (33, 17, 0)):
        g1 = ratio[np.arange(n) % len(ratio)].copy()
        g1[c, slot, 0] ^= np.uint64(1)
        with pytest.raises(_lib.B200Error) as err:
            pairing_check_many(ctx, g2, g1)
        assert err.value.code == _lib.B200_ERR_NOT_ON_CURVE and "check %d" % c in str(err.value)
        x = int.from_bytes(ratio[0, 0, 0:4].tobytes(), "little")
        g1 = ratio[np.arange(n) % len(ratio)].copy()
        g1[c, 0, 0:4] = np.frombuffer((x + Q).to_bytes(32, "little"), dtype="<u8")  # outside [0, q)
        with pytest.raises(_lib.B200Error) as err:
            pairing_check_many(ctx, g2, g1)
        assert err.value.code == _lib.B200_ERR_NOT_ON_CURVE and "check %d" % c in str(err.value)


# ---- verify_each on both sides of the switch --------------------------------------------------------------------------
LOG_N, NUM_INPUTS = 7, 4
LAYOUT = (5, 20, 6)


class Env:
    pass


@pytest.fixture(scope="module")
def env(ctx, srs_head, g2_raw):
    e = Env()
    e.ctx = ctx
    e.h, e.tau_h = g2_raw
    srs = rb.parse_ptau_file(ctx, srs_head, count=512).powers_of_g
    vals = [(0xC0DE + 31 * i) ** 5 % synth.R for i in range(LAYOUT[2])]
    circ = synth.synth_circuit(LOG_N, num_inputs=NUM_INPUTS, seed=2, check=True, link=(LAYOUT[0], LAYOUT[1], vals))
    pk = PlonkKzgSnark.preprocess(ctx, srs, LOG_N, NUM_INPUTS, circ.selectors, circ.perm, circ.k)
    proofs, hints = [], []
    for b in (20, 21):
        proof, hint = PlonkKzgSnark.prove_with_link_hint(ctx, pk, circ.wires, circ.pub_inputs, synth.splitmix_blinders(b))
        proofs.append(vm.PlonkItem(pk.k, pk.selector_comms, pk.sigma_comms, circ.pub_inputs, proof.to_array()))
        hints.append(hint)
    pk.free()
    lp, _ = link_proofs(ctx, srs, hints[0], hints[1], GroupLayout(*LAYOUT))
    link = vm.LinkItem(hints[0].linking_wire_comm, hints[1].linking_wire_comm, lp.to_array(), LAYOUT)
    pm, lm = vm.plonk_mutations(proofs[0]), vm.link_mutations(link)
    e.proofs = proofs + [m.item for cls in vm.CLASSES if any(x.cls == cls for x in pm)
                         for m in vm.representatives(pm, cls, 1)]
    e.links = [link] + [m.item for cls in vm.CLASSES if any(x.cls == cls for x in lm) for m in vm.representatives(lm, cls, 1)]
    e.proof_want = [single_plonk(e, it) for it in e.proofs]
    e.link_want = [single_link(e, it) for it in e.links]
    assert e.proof_want[:2] == [True, True] and not any(e.proof_want[2:])
    assert e.link_want[0] and not any(e.link_want[1:])
    return e


def _vk(e, it):
    return VerifyingKey(LOG_N, NUM_INPUTS, it.k, it.sel, it.sig, e.h, e.tau_h)


def single_plonk(e, it) -> bool:
    return PlonkKzgSnark.verify(_vk(e, it), it.pi, B200Proof.from_buffer_copy(it.proof.tobytes()))


def single_link(e, it) -> bool:
    return verify_link_proof(it.c1, it.c2, B200LinkProof.from_buffer_copy(it.lp.tobytes()), GroupLayout(*it.layout),
                             e.h, e.tau_h)


def _args(e, n_proofs, n_links):
    ps = [e.proofs[i % len(e.proofs)] for i in range(n_proofs)]
    ls = [e.links[i % len(e.links)] for i in range(n_links)]
    want = [e.proof_want[i % len(e.proofs)] for i in range(n_proofs)] + [e.link_want[i % len(e.links)] for i in range(n_links)]
    args = ([_vk(e, it) for it in ps], [it.pi for it in ps], [B200Proof.from_buffer_copy(it.proof.tobytes()) for it in ps],
            [(it.c1, it.c2, B200LinkProof.from_buffer_copy(it.lp.tobytes()), GroupLayout(*it.layout)) for it in ls])
    return args, want


@pytest.mark.parametrize("where", ["below", "above"])
def test_verify_each_equals_the_single_verifiers(env, where):
    e = env
    k = len(e.proofs) + len(e.links) if where == "below" else wave() + 1
    n_links = len(e.links) if where == "below" else k // 4
    args, want = _args(e, k - n_links, n_links)
    assert PlonkKzgSnark.verify_each(e.ctx, *args, g2=(e.h, e.tau_h)) == want


def test_pool_verification_job(env):
    e = env
    pool = ProverPool(0, workers=2)
    try:
        for k, n_links in ((1, 0), (1, 1), (16, 5)):
            args, want = _args(e, k - n_links, n_links)
            assert pool.wait(pool.submit_verify(*args, g2=(e.h, e.tau_h))) == want
            assert PlonkKzgSnark.verify_each(e.ctx, *args, g2=(e.h, e.tau_h)) == want
    finally:
        pool.close()
