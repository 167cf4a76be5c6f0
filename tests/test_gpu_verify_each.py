"""Per-item verification on the device (`b200_plonk_verify_each`, `PlonkKzgSnark.verify_each`): each proof and link
proof checked on its own with its own pairing must give, item by item, the answers of the single host verifiers, and
the verdicts of the batch verifier.  Proofs and links are those of tests/test_gpu_batch_verify.py (the device prover on
the reference's SRS head and its G2 pair)."""
import ctypes as C
import random

import numpy as np
import pytest

import verify_mutations as vm
from renegade_b200 import _lib
from renegade_b200.backend import B200LinkProof, B200Proof, GroupLayout, PlonkKzgSnark, VerifyingKey
from test_gpu_batch_verify import _tamper, env, proof_items, single_verdicts  # noqa: F401
from test_gpu_pairing_many import Q, _neg

pytestmark = pytest.mark.gpu

KINDS = ["eval_bit", "swap_comms", "pub_input", "wrong_vk", "off_curve", "link_layout"]


def each(e, items, links):
    return PlonkKzgSnark.verify_each(e.ctx, [i[0] for i in items], [i[1] for i in items], [i[2] for i in items], links,
                                     g2=(e.h, e.tau_h))


def _bad_proof(proof, bit=0):
    p = B200Proof.from_buffer_copy(bytes(proof))
    p.wires_evals[3][0] ^= 1 << bit
    return p


def test_mixed_batch(env):
    e = env
    order = [2, 0, 4, 1, 6, 3, 5, 7] + [4, 5] * 18 + [0, 2]
    items = proof_items(e, order)
    assert sum(it[0].num_inputs or 1 for it in items) > 4096
    links = e.links + e.links[:2]
    assert each(e, items, links) == [True] * (len(items) + len(links))
    assert single_verdicts(e, items[:8], links) == [True] * (8 + len(links))


@pytest.mark.parametrize("kind", KINDS)
def test_every_tampering_kind(env, kind):
    e = env
    items = proof_items(e, [2, 0, 4, 3, 6, 1, 5, 7, 3])
    n_links = len(e.links)
    positions = [0, n_links // 2, n_links - 1] if kind == "link_layout" else [0, len(items) // 2, len(items) - 1]
    for pos in positions:
        its, lks = _tamper(e, kind, items, e.links, pos)
        want = single_verdicts(e, its, lks)
        assert want.count(False) == 1, (kind, pos)
        assert each(e, its, lks) == want, (kind, pos)


def test_every_item_bad_and_alternate_items_bad(env):
    e = env
    items = proof_items(e, [0, 1, 2, 3, 6, 7])
    links = [(a, b, lp, GroupLayout(lay.alignment, lay.offset + 1, lay.size)) for a, b, lp, lay in e.links]
    bad = [(vk, pi, _bad_proof(p)) for vk, pi, p in items]
    want = single_verdicts(e, bad, links)
    assert want == [False] * (len(bad) + len(links))
    assert each(e, bad, links) == want
    alt = [bad[i] if i % 2 else items[i] for i in range(len(items))]
    alt_links = [links[i] if i % 2 == 0 else e.links[i] for i in range(len(e.links))]
    want = single_verdicts(e, alt, alt_links)
    assert want == [i % 2 == 0 for i in range(len(items))] + [i % 2 == 1 for i in range(len(e.links))]
    assert each(e, alt, alt_links) == want


def test_links_only_proofs_only_and_small_sizes(env):
    e = env
    assert PlonkKzgSnark.verify_each(e.ctx, [], [], [], e.links, g2=(e.h, e.tau_h)) == [True] * len(e.links)
    assert each(e, proof_items(e, [0, 2, 4]), []) == [True] * 3
    assert PlonkKzgSnark.verify_each(e.ctx, [], [], [], [], g2=(e.h, e.tau_h)) == []
    assert each(e, proof_items(e, [5]), []) == [True]
    assert each(e, [], [e.links[1]]) == [True]
    vk, pi, p = proof_items(e, [5])[0]
    assert each(e, [(vk, pi, _bad_proof(p))], []) == [False]
    # a wrong public-input count is a False verdict, as for the single verifier
    vk2, pi2, p2 = proof_items(e, [2])[0]
    assert each(e, [proof_items(e, [0])[0], (vk2, pi2[:-1], p2)], []) == [True, False]


def test_openings_that_cancel_are_each_rejected(env):
    """Link items with openings pi + G and pi - G: their unweighted sum satisfies the link equation, but each item is
    checked on its own here, with no combination at all."""
    e = env
    a, b, lp, lay = e.links[0]
    mont = lambda v: np.frombuffer(((v << 256) % Q).to_bytes(32, "little"), dtype="<u8")
    g = np.concatenate([mont(1), mont(2)]).astype(np.uint64)
    pi = np.array(lp.opening_proof, dtype=np.uint64)
    plus, _ = e.ctx.g1_sum_affine(np.stack([pi, g]))
    minus, _ = e.ctx.g1_sum_affine(np.stack([pi, _neg(g)]))
    pair = []
    for op in (plus, minus):
        x = B200LinkProof.from_buffer_copy(bytes(lp))
        x.opening_proof[:] = [int(v) for v in op]
        pair.append((a, b, x, lay))
    assert single_verdicts(e, [], pair) == [False, False]
    assert PlonkKzgSnark.verify_each(e.ctx, [], [], [], pair, g2=(e.h, e.tau_h)) == [False, False]
    assert each(e, proof_items(e, [0, 1]), [e.links[1]] + pair + [e.links[2]]) == [True, True, True, False, False, True]


def test_identity_selector_commitment(env):
    """A key with the identity as one selector commitment (tests/test_gpu_batch_verify.py builds the same key)."""
    from renegade_b200 import synth
    e = env
    log_n, ni = 7, 4
    circ = synth.synth_circuit(log_n, num_inputs=ni, seed=21, check=True)
    sel = circ.selectors_int
    for r in range(circ.n):
        if sel[synth.Q_ECC][r]:
            w = [circ.wires_int[j][r] for j in range(5)]
            sel[synth.Q_C][r] = (sel[synth.Q_C][r] + sel[synth.Q_ECC][r] * w[0] * w[1] * w[2] * w[3] * w[4]) % synth.R
            sel[synth.Q_ECC][r] = 0
    selectors = np.stack([synth.to_mont_array(col) for col in sel])
    pk = PlonkKzgSnark.preprocess(e.ctx, e.srs, log_n, ni, selectors, circ.perm, circ.k)
    try:
        assert not pk.selector_comms[synth.Q_ECC].any()
        vk = VerifyingKey.from_proving_key(pk, e.h, e.tau_h)
        proof, _ = PlonkKzgSnark.prove_with_link_hint(e.ctx, pk, circ.wires, circ.pub_inputs, synth.splitmix_blinders(5))
        items = [(vk, circ.pub_inputs, proof)] + proof_items(e, [2, 3]) + [(vk, circ.pub_inputs, _bad_proof(proof))]
        want = single_verdicts(e, items, [])
        assert want == [True, True, True, False]
        assert each(e, items, []) == want
    finally:
        pk.free()


def test_every_mutation_is_rejected(env):
    """Every single-field mutation of verify_mutations.py of a 4-input proof item and of a link item, in one call
    beside the honest items: each mutation rejected, each honest item accepted."""
    e = env
    pk, _ = e.keys[1]
    _, pi, proof, _ = e.proofs[2]
    honest = vm.PlonkItem(pk.k, pk.selector_comms, pk.sigma_comms, pi, proof.to_array())
    a, b, lp, lay = e.links[0]
    honest_link = vm.LinkItem(a, b, lp.to_array(), (lay.alignment, lay.offset, lay.size))
    pmuts = [m.item for m in vm.plonk_mutations(honest)]
    lmuts = [m.item for m in vm.link_mutations(honest_link)]
    proofs = [honest] + pmuts + [honest]
    links = [honest_link] + lmuts + [honest_link]
    vks = [VerifyingKey(pk.log_n, pk.num_inputs, it.k, it.sel, it.sig, e.h, e.tau_h) for it in proofs]
    lks = [(it.c1, it.c2, B200LinkProof.from_buffer_copy(it.lp.tobytes()), GroupLayout(*it.layout)) for it in links]
    got = PlonkKzgSnark.verify_each(e.ctx, vks, [it.pi for it in proofs],
                                    [B200Proof.from_buffer_copy(it.proof.tobytes()) for it in proofs], lks,
                                    g2=(e.h, e.tau_h))
    assert got == [True] + [False] * len(pmuts) + [True] + [True] + [False] * len(lmuts) + [True]


def test_half_of_4096_tampered(env):
    """k = 4096 with a seeded half of the items tampered: the batch verifier's verdicts over all items, and the single
    host verifiers' on a seeded sample of 256."""
    e = env
    base = proof_items(e, [0, 1, 2, 3, 6, 7])
    rnd = random.Random(4096)
    bad = set(rnd.sample(range(4096), 2048))
    items = []
    for i in range(4096):
        vk, pi, p = base[i % len(base)]
        items.append((vk, pi, _bad_proof(p, i % 64) if i in bad else p))
    got = each(e, items, [])
    assert got == [i not in bad for i in range(4096)]
    ok, batch_verdicts = PlonkKzgSnark.batch_verify(e.ctx, [i[0] for i in items], [i[1] for i in items],
                                                    [i[2] for i in items], g2=(e.h, e.tau_h))
    assert not ok and got == batch_verdicts
    sample = sorted(rnd.sample(range(4096), 256))
    assert [got[i] for i in sample] == single_verdicts(e, [items[i] for i in sample], [])


def test_argument_errors(env):
    e = env
    vk, pi, p = proof_items(e, [2])[0]
    other = VerifyingKey(vk.log_n, vk.num_inputs, vk.k, vk.selector_comms, vk.sigma_comms, e.tau_h, e.h)
    with pytest.raises(ValueError):
        PlonkKzgSnark.verify_each(e.ctx, [vk, other], [pi] * 2, [p] * 2)
    lib = e.ctx._lib
    h = e.h.ctypes.data_as(C.c_void_p)
    out = (C.c_uint8 * 1)()
    assert lib.b200_plonk_verify_each(None, None, 0, None, 0, None, 0, h, h, out) == _lib.B200_ERR_INVALID
    assert lib.b200_plonk_verify_each(e.ctx._h, None, 0, None, 1, None, 0, h, h, out) == _lib.B200_ERR_INVALID
    assert lib.b200_plonk_verify_each(e.ctx._h, None, 0, None, 0, None, 0, None, h, out) == _lib.B200_ERR_INVALID
    assert lib.b200_plonk_verify_each(e.ctx._h, None, 0, None, 0, None, 0, h, h, None) == _lib.B200_OK  # no items
    # a link with size 0, and an off-curve G2 point, as for the batch verifier
    a, b, lp, lay = e.links[0]
    with pytest.raises(_lib.B200Error) as err:
        PlonkKzgSnark.verify_each(e.ctx, [], [], [], [(a, b, lp, GroupLayout(lay.alignment, lay.offset, 0))],
                                  g2=(e.h, e.tau_h))
    assert err.value.code == _lib.B200_ERR_INVALID and "verify_each" in str(err.value)
    bad_h = np.array(e.h, dtype=np.uint64)
    bad_h[0] ^= np.uint64(1)
    with pytest.raises(_lib.B200Error) as err:
        PlonkKzgSnark.verify_each(e.ctx, [], [], [], [e.links[0]], g2=(bad_h, e.tau_h))
    assert err.value.code == _lib.B200_ERR_NOT_ON_CURVE
