"""GPU parity of the prover's CUDA-graph replay: from the second proof of a key on a context every prover segment is one
graph submission (csrc/plonk.cu run_segment).  The bytes must not depend on how the launches were submitted: eager,
captured-and-launched, replayed, recaptured after a buffer moved — all equal the CPU restatement's proof for the same
witness and blinders."""
import numpy as np
import pytest

from renegade_b200 import synth
from renegade_b200._lib import B200Error
from renegade_b200.backend import PlonkKzgSnark

pytestmark = pytest.mark.gpu

TAU = 0x2f1a6c0b5d3e49788a9bc0d1e2f30415263748596a7b8c9dae0f1f2e3d4c5b6a
SEGMENTS = 7  # graph submissions per replayed proof


def make(ctx, oracle, pyoracle, log_n, seed):
    n = 1 << log_n
    circ = synth.synth_circuit(log_n, num_inputs=5, seed=seed, check=(log_n <= 10))
    tau = oracle.int_to_limbs(pyoracle.to_mont(TAU % pyoracle.R, pyoracle.R))
    srs = oracle.srs_from_tau(tau, n + 3)
    bases = ctx.load_bases(srs)
    pk = PlonkKzgSnark.preprocess(ctx, bases, log_n, circ.num_inputs, circ.selectors, circ.perm, circ.k)
    opk = oracle.plonk_preprocess(log_n, circ.selectors, circ.perm, circ.k, srs)
    return circ, srs, bases, pk, opk


def check(ctx, oracle, log_n, circ, srs, pk, opk, blind_seed):
    bl = synth.splitmix_blinders(blind_seed)
    proof, hint, ch = PlonkKzgSnark.prove_with_link_hint(ctx, pk, circ.wires, circ.pub_inputs, bl, want_challenges=True)
    rc, oproof, och, olink = oracle.plonk_prove(log_n, circ.num_inputs, circ.k, opk, circ.wires, circ.pub_inputs, bl, srs, True)
    assert rc == 0
    assert bytes(proof) == bytes(oproof), "blinders %d" % blind_seed
    assert (ch.reshape(-1) == np.frombuffer(bytes(och), dtype=np.uint64)).all()
    assert (hint.linking_wire_poly == olink).all()


@pytest.mark.parametrize("log_n", [4, 9, 13])
def test_replayed_proofs_equal_the_oracle(ctx, oracle, pyoracle, log_n):
    circ, srs, bases, pk, opk = make(ctx, oracle, pyoracle, log_n, seed=300 + log_n)
    ctx.use_graphs(True)
    g0 = ctx.graph_launches()
    k = []
    for i in range(5):  # eager, capture + launch, replay, replay, replay — different blinders every time
        k0 = ctx.kernel_launches()
        check(ctx, oracle, log_n, circ, srs, pk, opk, 9000 + 17 * i + log_n)
        k.append(ctx.kernel_launches() - k0)
    assert ctx.graph_launches() - g0 == 4 * SEGMENTS
    assert len(set(k)) == 1, k  # the same kernels run however they were submitted
    pk.free()
    bases.free()


def test_two_keys_interleaved_and_recapture_after_growth(ctx, oracle, pyoracle):
    """A small key's graphs are captured, then a larger key grows the context's buffers (they move): the small key's
    graphs are stale and must be captured again, not replayed onto freed memory."""
    ctx.use_graphs(True)
    a = make(ctx, oracle, pyoracle, 7, seed=41)
    check(ctx, oracle, 7, a[0], a[1], a[3], a[4], 1)   # eager
    check(ctx, oracle, 7, a[0], a[1], a[3], a[4], 2)   # captured
    check(ctx, oracle, 7, a[0], a[1], a[3], a[4], 3)   # replayed
    b = make(ctx, oracle, pyoracle, 14, seed=42)       # larger than anything this file used so far
    for i in range(3):
        check(ctx, oracle, 14, b[0], b[1], b[3], b[4], 10 + i)
        check(ctx, oracle, 7, a[0], a[1], a[3], a[4], 20 + i)
    for x in (a, b):
        x[3].free()
        x[2].free()


def test_unsatisfied_witness_in_a_replayed_round(ctx, oracle, pyoracle):
    log_n = 8
    circ, srs, bases, pk, opk = make(ctx, oracle, pyoracle, log_n, seed=77)
    ctx.use_graphs(True)
    for i in range(3):
        check(ctx, oracle, log_n, circ, srs, pk, opk, 50 + i)
    bad = circ.wires.copy()
    bad[4, circ.num_inputs + 3] = bad[4, circ.num_inputs + 4]
    with pytest.raises(B200Error) as e:
        PlonkKzgSnark.prove_with_link_hint(ctx, pk, bad, circ.pub_inputs, synth.splitmix_blinders(1))
    assert e.value.code == -7
    check(ctx, oracle, log_n, circ, srs, pk, opk, 60)  # the context keeps proving
    pk.free()
    bases.free()


def test_graphs_off_is_eager(ctx, oracle, pyoracle):
    log_n = 6
    circ, srs, bases, pk, opk = make(ctx, oracle, pyoracle, log_n, seed=12)
    ctx.use_graphs(False)
    try:
        g0 = ctx.graph_launches()
        for i in range(3):
            check(ctx, oracle, log_n, circ, srs, pk, opk, 70 + i)
        assert ctx.graph_launches() == g0
    finally:
        ctx.use_graphs(True)
    pk.free()
    bases.free()


def test_link_proofs_replayed(ctx, oracle, pyoracle):
    """A link proof's launches depend on (SRS, lengths, layout) only: two graph segments from the second call on.  Different
    witnesses (hence different eta) every time; each must equal the oracle's link proof; a wrong layout is still refused."""
    from renegade_b200.backend import GroupLayout, link_proofs
    py = pyoracle
    layout = GroupLayout(alignment=7, offset=20, size=9)
    tau = oracle.int_to_limbs(py.to_mont(TAU % py.R, py.R))
    srs = oracle.srs_from_tau(tau, (1 << 10) + 3)
    bases = ctx.load_bases(srs)
    ctx.use_graphs(True)
    g0 = ctx.graph_launches()
    kept = []  # every round's hints stay alive: each call reads polynomials at addresses no earlier call used
    for rnd in range(4):
        vals = [(i * 0x9E3779B97F4A7C15 + 777 * rnd + 5) % py.R for i in range(layout.size)]
        hints = []
        for log_n, seed in ((9, 3), (10, 4)):  # a fresh key every round (the selectors may depend on the pinned values)
            circ = synth.synth_circuit(log_n, num_inputs=5, seed=seed, check=True, link=(layout.alignment, layout.offset, vals))
            pk = PlonkKzgSnark.preprocess(ctx, bases, log_n, circ.num_inputs, circ.selectors, circ.perm, circ.k)
            _, hint = PlonkKzgSnark.prove_with_link_hint(ctx, pk, circ.wires, circ.pub_inputs, synth.splitmix_blinders(seed + rnd))
            pk.free()
            hints.append(hint)
        kept.append(hints)
        lp, eta = link_proofs(ctx, bases, hints[0], hints[1], layout)
        rc, olp, oeta = oracle.plonk_link(hints[0].linking_wire_poly, hints[1].linking_wire_poly, hints[0].linking_wire_comm,
                                          hints[1].linking_wire_comm, layout.alignment, layout.offset, layout.size, srs)
        assert rc == 0
        assert (lp.to_array() == olp.to_array()).all() and (eta == oeta).all(), rnd
        if rnd == 2:  # a REPLAYED first segment must still flag an inexact division: last round's second polynomial
            with pytest.raises(B200Error) as err:
                link_proofs(ctx, bases, hints[0], prev[1], layout)
            assert err.value.code == -7
            with pytest.raises(B200Error) as err:  # and a layout the proofs do not share (a key of its own: eager)
                link_proofs(ctx, bases, hints[0], hints[1], GroupLayout(layout.alignment, layout.offset + 1, layout.size))
            assert err.value.code == -7
        prev = hints
    # rounds 1..3: the link proof's 2 segments replayed, plus the first segment of the refused call; round 0 eager; the
    # proofs use fresh keys (eager)
    assert ctx.graph_launches() - g0 == 3 * 2 + 1
    bases.free()
