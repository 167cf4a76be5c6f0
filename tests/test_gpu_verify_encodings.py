"""The batch verifier (`b200_plonk_batch_verify`) on the mutation matrix of `verify_mutations.py`: every proof point,
evaluation and public input, every verifying-key field, every part of a link proof and its layout, moved outside the
field (v + p, the largest v + m p below 2^256, 2^256 - 1) or to a wrong canonical value.  Each verdict must equal the
single host verifier's (tests/test_verify_encodings_cpu.py holds those to "rejected"): an encoding outside [0, p)
that reached the device's transcript, multipliers and MSM as if it were its residue would be accepted there.

Only wrong values are passed: every buffer has its honest size, and the MSM's digits stay inside their buckets for
any 256-bit scalar.  Proofs come from the device prover on the reference's SRS head and its G2 pair."""
import numpy as np
import pytest

import renegade_b200 as rb
import verify_mutations as vm
from renegade_b200 import _lib, synth
from renegade_b200.backend import (B200LinkProof, B200Proof, GroupLayout, PlonkKzgSnark, VerifyingKey, link_proofs,
                                   verify_link_proof)

pytestmark = pytest.mark.gpu

LOG_N, NUM_INPUTS = 7, 4
LAYOUT = (5, 20, 6)  # alignment, offset, size
B200_ERR_NOT_ON_CURVE = -5


class Env:
    pass


@pytest.fixture(scope="module")
def env(ctx, srs_head, g2_raw):
    e = Env()
    e.ctx = ctx
    e.h, e.tau_h = g2_raw
    srs = rb.parse_ptau_file(ctx, srs_head, count=512).powers_of_g
    vals = [(0xC0DE + 31 * i) ** 5 % synth.R for i in range(LAYOUT[2])]
    e.proofs, hints = [], []
    for log_n, ni, seed, blinders in ((LOG_N, NUM_INPUTS, 2, (20, 21)), (6, 0, 1, (22,))):
        circ = synth.synth_circuit(log_n, num_inputs=ni, seed=seed, check=True, link=(LAYOUT[0], LAYOUT[1], vals))
        pk = PlonkKzgSnark.preprocess(ctx, srs, log_n, ni, circ.selectors, circ.perm, circ.k)
        for b in blinders:
            proof, hint = PlonkKzgSnark.prove_with_link_hint(ctx, pk, circ.wires, circ.pub_inputs,
                                                             synth.splitmix_blinders(b))
            hints.append(hint)
            if log_n == LOG_N:
                e.proofs.append(vm.PlonkItem(pk.k, pk.selector_comms, pk.sigma_comms, circ.pub_inputs, proof.to_array()))
        pk.free()
    e.links = []
    for a in (0, 1):  # the 2^6 proof linked to each 2^7 proof
        lp, _ = link_proofs(ctx, srs, hints[2], hints[a], GroupLayout(*LAYOUT))
        e.links.append(vm.LinkItem(hints[2].linking_wire_comm, hints[a].linking_wire_comm, lp.to_array(), LAYOUT))
    e.plonk_muts = vm.plonk_mutations(e.proofs[0])
    e.link_muts = vm.link_mutations(e.links[0])
    # the single verifiers reject every mutation and accept the honest items
    assert [single_plonk(e, p) for p in e.proofs] == [True, True]
    assert [single_link(e, lk) for lk in e.links] == [True, True]
    assert not any(single_plonk(e, m.item) for m in e.plonk_muts)
    assert not any(single_link(e, m.item) for m in e.link_muts)
    return e


def _vk(e, it, h=None, tau_h=None):
    return VerifyingKey(LOG_N, NUM_INPUTS, it.k, it.sel, it.sig, e.h if h is None else h, e.tau_h if tau_h is None else tau_h)


def single_plonk(e, it) -> bool:
    return PlonkKzgSnark.verify(_vk(e, it), it.pi, B200Proof.from_buffer_copy(it.proof.tobytes()))


def single_link(e, it) -> bool:
    return verify_link_proof(it.c1, it.c2, B200LinkProof.from_buffer_copy(it.lp.tobytes()), GroupLayout(*it.layout),
                             e.h, e.tau_h)


def batch(e, proofs, links, h=None, tau_h=None):
    vks = [_vk(e, it, h, tau_h) for it in proofs]
    lks = [(it.c1, it.c2, B200LinkProof.from_buffer_copy(it.lp.tobytes()), GroupLayout(*it.layout)) for it in links]
    g2 = (e.h if h is None else h, e.tau_h if tau_h is None else tau_h)
    return PlonkKzgSnark.batch_verify(e.ctx, vks, [it.pi for it in proofs],
                                      [B200Proof.from_buffer_copy(it.proof.tobytes()) for it in proofs], lks, g2=g2)


def test_honest_batch_is_accepted(env):
    e = env
    ok, verdicts = batch(e, [e.proofs[0], e.proofs[1], e.proofs[0]], e.links)
    assert ok and verdicts == [True] * 5


def test_one_batch_of_everything(env):
    """All mutations and the honest items in one call: nothing accepted, each verdict the single verifier's."""
    e = env
    muts = [m.item for m in e.plonk_muts]
    half = len(muts) // 2
    proofs = [e.proofs[0]] + muts[:half] + [e.proofs[1]] + muts[half:] + [e.proofs[0]]
    links = [e.links[0]] + [m.item for m in e.link_muts] + [e.links[1]]
    want = ([True] + [False] * half + [True] + [False] * (len(muts) - half) + [True] +
            [True] + [False] * len(e.link_muts) + [True])
    ok, verdicts = batch(e, proofs, links)
    assert not ok and len(verdicts) == len(want)
    labels = (["honest"] + [m.label for m in e.plonk_muts[:half]] + ["honest"] + [m.label for m in e.plonk_muts[half:]] +
              ["honest", "honest"] + [m.label for m in e.link_muts] + ["honest"])
    wrong = [labels[i] for i in range(len(want)) if verdicts[i] != want[i]]
    assert wrong == []


@pytest.mark.parametrize("cls", vm.CLASSES)
def test_each_class_first_middle_last(env, cls):
    """One mutation of the class among honest items, first, in the middle and last of its list (proofs or links)."""
    e = env
    reps = vm.representatives(e.plonk_muts + e.link_muts, cls)
    for place, m in zip(("first", "middle", "last"), reps):
        is_link = isinstance(m.item, vm.LinkItem)
        honest = list(e.links) + [e.links[0]] if is_link else [e.proofs[0], e.proofs[1], e.proofs[0]]
        pos = {"first": 0, "middle": len(honest) // 2, "last": len(honest)}[place]
        group = honest[:pos] + [m.item] + honest[pos:]
        proofs, links = ([e.proofs[1]], group) if is_link else (group, [e.links[1]])
        want = [single_plonk(e, it) for it in proofs] + [single_link(e, it) for it in links]
        assert want.count(False) == 1, m.label
        ok, verdicts = batch(e, proofs, links)
        assert not ok, (m.label, place)
        assert verdicts == want, (m.label, place)


def test_non_canonical_g2_is_refused(env):
    """A G2 record with a coordinate >= q is off the curve for the batch verifier too: B200_ERR_NOT_ON_CURVE."""
    e = env
    for which in ("h", "tau_h"):
        rec = getattr(e, which)
        for j in range(4):
            for enc in vm.out_of_field(vm.to_int(rec[4 * j:4 * j + 4]), vm.Q).values():
                bad = np.array(rec, dtype=np.uint64)
                bad[4 * j:4 * j + 4] = vm.to_words(enc)
                with pytest.raises(_lib.B200Error) as err:
                    batch(e, [e.proofs[0]], [e.links[0]], **{which: bad})
                assert err.value.code == B200_ERR_NOT_ON_CURVE, (which, j, enc)
