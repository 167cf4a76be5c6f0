"""GPU parity: proof linking (`PlonkKzgSnark::link_proofs`) on the device vs the CPU restatement.
Two circuits of different sizes share a link group (same values on the same 2^alignment-th roots of
unity in wire 0); their proofs' linking hints are linked on the device; the link proof is
byte-identical to the oracle's and accepted by the restated link verifier; a mismatching group is
rejected."""
import numpy as np
import pytest

from renegade_b200 import synth
from renegade_b200.backend import GroupLayout, PlonkKzgSnark, link_proofs

pytestmark = pytest.mark.gpu

TAU = 0x1b0a7c3d5e9f00112233445566778899aabbccddeeff0123456789abcdef0f1e


def test_link_two_circuits(ctx, oracle, pyoracle):
    py = pyoracle
    layout = GroupLayout(alignment=8, offset=40, size=12)
    vals = [(i * 0x9E3779B97F4A7C15 + 12345) % py.R for i in range(layout.size)]
    tau = oracle.int_to_limbs(py.to_mont(TAU % py.R, py.R))
    srs = oracle.srs_from_tau(tau, (1 << 11) + 3)
    bases = ctx.load_bases(srs)
    hints = []
    for log_n, seed in ((10, 3), (11, 4)):
        circ = synth.synth_circuit(log_n, num_inputs=5, seed=seed, check=True,
                                   link=(layout.alignment, layout.offset, vals))
        # the link values sit on wire 0 at the rows of the 2^alignment-th roots of unity
        for i, v in enumerate(vals):
            assert circ.wires_int[0][(layout.offset + i) << (log_n - layout.alignment)] == v
        pk = PlonkKzgSnark.preprocess(ctx, bases, log_n, circ.num_inputs, circ.selectors, circ.perm, circ.k)
        proof, hint = PlonkKzgSnark.prove_with_link_hint(ctx, pk, circ.wires, circ.pub_inputs, synth.splitmix_blinders(seed))
        opk = {"selector_comms": pk.selector_comms, "sigma_comms": pk.sigma_comms}
        assert oracle.plonk_verify_known_tau(log_n, circ.num_inputs, circ.k, opk, circ.pub_inputs,
                                             oracle.PlonkProof.from_buffer_copy(bytes(proof)), tau)
        hints.append(hint)
    lp, eta = link_proofs(ctx, bases, hints[0], hints[1], layout)
    rc, olp, oeta = oracle.plonk_link(hints[0].linking_wire_poly, hints[1].linking_wire_poly, hints[0].linking_wire_comm,
                                      hints[1].linking_wire_comm, layout.alignment, layout.offset, layout.size, srs)
    assert rc == 0
    assert (lp.to_array() == olp.to_array()).all() and (eta == oeta).all()
    assert oracle.plonk_link_verify_known_tau(hints[0].linking_wire_comm, hints[1].linking_wire_comm, layout.alignment,
                                              layout.offset, layout.size, oracle.LinkProof.from_buffer_copy(bytes(lp)), tau)
    # a group the two proofs do NOT share (one row further) must not verify
    wrong = GroupLayout(layout.alignment, layout.offset + 1, layout.size)
    import pytest
    from renegade_b200._lib import B200Error
    with pytest.raises(B200Error) as err:      # the prover refuses: a division by the group's roots is not exact
        link_proofs(ctx, bases, hints[0], hints[1], wrong)
    assert err.value.code == -7
    # the refused call zeroes the caller's proof buffer and leaves its eta buffer alone
    import ctypes as C
    from renegade_b200.backend import B200LinkProof
    a1, a2, c1, c2 = (np.ascontiguousarray(x, dtype=np.uint64) for x in (hints[0].linking_wire_poly, hints[1].linking_wire_poly,
                                                                         hints[0].linking_wire_comm, hints[1].linking_wire_comm))
    junk, eta_buf = B200LinkProof.from_buffer_copy(b"\xa5" * C.sizeof(B200LinkProof)), np.full(4, 7, dtype=np.uint64)
    vp = lambda a: a.ctypes.data_as(C.c_void_p)  # noqa: E731
    assert (ctx._lib.b200_plonk_link(ctx._h, bases._h, vp(a1), a1.size // 4, vp(a2), a2.size // 4, vp(c1), vp(c2), wrong.alignment,
                                     wrong.offset, wrong.size, C.byref(junk), vp(eta_buf)) == -7
            and bytes(junk) == bytes(C.sizeof(B200LinkProof)) and (eta_buf == 7).all())
    rc, _, _ = oracle.plonk_link(hints[0].linking_wire_poly, hints[1].linking_wire_poly, hints[0].linking_wire_comm,
                                 hints[1].linking_wire_comm, wrong.alignment, wrong.offset, wrong.size, srs)
    assert rc == 2
    # and the honest proof does not verify under the wrong layout
    assert not oracle.plonk_link_verify_known_tau(hints[0].linking_wire_comm, hints[1].linking_wire_comm, wrong.alignment,
                                                  wrong.offset, wrong.size, oracle.LinkProof.from_buffer_copy(bytes(lp)), tau)
    # the context stays usable after the refusal
    lp3, _ = link_proofs(ctx, bases, hints[0], hints[1], layout)
    assert (lp3.to_array() == lp.to_array()).all()
