"""The verifier sweep of `verify_sweep.py` (every domain 2^2 ... 2^17, 0, 1, 5 and all public inputs, every link layout,
each with its tampered twins) checked without a device: every item is what the builder says it is, the host single
verifiers and the oracle's known-tau verifiers give every item the same verdict, and it is the expected one.  And the
link verifier's layout rule: a group of more roots than its 2^alignment subgroup holds is refused before Z_D is formed,
so a caller's size cannot keep the verifier busy for 2^64 products."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import verify_sweep as vs
from renegade_b200 import _lib
from renegade_b200.backend import B200LinkProof, B200Proof, GroupLayout, PlonkKzgSnark, VerifyingKey, verify_link_proof


@pytest.fixture(scope="module")
def sweep(oracle):
    return vs.build(oracle)


def _int(limbs) -> int:
    return int.from_bytes(np.asarray(limbs, dtype=np.uint64).tobytes(), "little")


def test_proofs_are_what_the_builder_claims(sweep):
    sw = sweep
    honest = {it.name: it for it in sw.proofs if it.kind == "honest"}
    assert sorted((it.log_n, it.num_inputs) for it in honest.values()) == sorted(vs.shapes())
    assert {lg for lg, _ in vs.shapes()} == set(range(2, 18))
    twins = {}
    for it in sw.proofs:
        assert it.want == (it.kind == "honest"), it.name
        if it.kind == "honest":
            assert it.key == (it.log_n, it.num_inputs) and it.pi.shape == (it.num_inputs, 4)
            continue
        base = honest[it.name.rsplit(":", 1)[0]]
        twins.setdefault(base.name, set()).add(it.kind)
        diff = np.nonzero(it.proof != base.proof)[0]
        if it.kind == "eval_bit":
            assert len(diff) == 1 and 104 <= diff[0] < 144 and it.key == base.key and (it.pi == base.pi).all()
            assert bin(int(it.proof[diff[0]] ^ base.proof[diff[0]])).count("1") == 1
            e = 104 + (diff[0] - 104) // 4 * 4
            assert _int(it.proof[e:e + 4]) < vs.R  # a canonical value, not an encoding outside the field
        elif it.kind == "last_input":
            assert len(diff) == 0 and it.key == base.key
            assert (it.pi[:-1] == base.pi[:-1]).all() and _int(it.pi[-1]) == (_int(base.pi[-1]) + vs.MONT % vs.R) % vs.R
        elif it.kind == "swap_wires":
            assert list(diff) == list(range(16)) and (it.proof[:8] == base.proof[8:16]).all()
            assert (it.proof[8:16] == base.proof[:8]).all() and it.key == base.key
        else:
            assert it.kind == "next_key" and len(diff) == 0 and it.key[1] == base.num_inputs
            assert it.key[0] == (base.log_n + 1 if base.log_n < 17 else 16)
    for name, it in honest.items():
        want = {"eval_bit", "swap_wires"} | ({"last_input"} if it.num_inputs else set())
        want |= {"next_key"} if it.num_inputs != 1 << it.log_n else set()
        assert twins[name] == want, name


def test_links_are_what_the_builder_claims(sweep, oracle):
    import link_layouts as ll
    sw = sweep
    assert len(sw.links) == 3 * len(ll.CASES)
    for c in ll.CASES:
        items = {it.kind: it for it in sw.links if it.case is c}
        h, s, w = items["honest"], items["shifted"], items["swapped"]
        assert h.layout == (c.alignment, c.offset, c.size) and s.layout == (c.alignment, c.offset + 1, c.size)
        assert (s.c1 == h.c1).all() and (w.c1 == h.c2).all() and (w.c2 == h.c1).all() and (w.lp == h.lp).all()
        assert (h.c1 == h.c2).all() == c.identical
        assert h.want and s.want == (c.identical or c.size == 1 << c.alignment) and w.want == c.identical


def test_every_warp_pair_kind_across_sizes(sweep):
    """pairs (2i, 2i+1) share a warp: honest/tampered, tampered/honest and honest/honest each at several sizes"""
    sw = sweep
    assert len(sw.proofs) % 2 == 0 and len(sw.links) % 2 == 0
    for items in (sw.proofs, sw.links):
        kinds = vs.pair_kinds([it.want for it in items])
        for k in ("HT", "TH", "HH"):
            sizes = {getattr(items[2 * i], "log_n", None) or items[2 * i].case.name for i, x in enumerate(kinds) if x == k}
            assert len(sizes) >= 3, (k, sizes)
    # the accepted items of the equal-polynomial link have the identity as their opening, so as a pairing operand: one
    # in the lower and one in the upper group of a warp
    assert {i % 2 for i, it in enumerate(sw.links) if it.case.identical and it.want} == {0, 1}


@pytest.mark.parametrize("log_n", list(range(2, 18)))
def test_host_and_oracle_verdicts_are_the_expected_ones(sweep, oracle, log_n):
    sw = sweep
    items = [it for it in sw.proofs if it.log_n == log_n]
    assert items
    for it in items:
        lg, ni, k, sel, sig = vs.vk_parts(sw, it)
        vk = VerifyingKey(lg, ni, k, sel, sig, sw.h, sw.tau_h)
        host = PlonkKzgSnark.verify(vk, it.pi, B200Proof.from_buffer_copy(it.proof.tobytes()))
        orc = oracle.plonk_verify_known_tau(lg, ni, k, sw.keys[it.key].pk, it.pi,
                                            oracle.PlonkProof.from_buffer_copy(it.proof.tobytes()), sw.tau)
        assert host == orc == it.want, it.name


def test_link_verdicts_are_the_expected_ones(sweep, oracle):
    sw = sweep
    for it in sw.links:
        host = verify_link_proof(it.c1, it.c2, B200LinkProof.from_buffer_copy(it.lp.tobytes()), GroupLayout(*it.layout),
                                 sw.h, sw.tau_h)
        orc = oracle.plonk_link_verify_known_tau(it.c1, it.c2, *it.layout, oracle.LinkProof.from_buffer_copy(it.lp.tobytes()),
                                                 sw.tau)
        assert host == orc == it.want, it.name


# ---- the layout rule of the host link verifier ------------------------------------------------------------------------
_PROBE = r"""
import ctypes as C, json, sys
import numpy as np
from renegade_b200 import _lib
lib = _lib.load()
g2 = np.frombuffer(open(sys.argv[1], "rb").read(), dtype=np.uint64)
h, tau_h = g2[:16].copy(), g2[16:32].copy()
zero = np.zeros(8, dtype=np.uint64)
p = lambda a: a.ctypes.data_as(C.c_void_p)  # noqa: E731
out = []
for a, size in json.loads(sys.argv[2]):
    ok, proof = C.c_int(7), (C.c_uint64 * 16)()
    rc = lib.b200_plonk_verify_link(p(zero), p(zero), a, 5, size, proof, p(h), p(tau_h), C.byref(ok))
    out.append([rc, ok.value])
    print(json.dumps(out), flush=True)
"""


def test_host_link_verifier_refuses_groups_larger_than_their_subgroup(tmp_path):
    """size 2^a + 1 and 2^63 are B200_ERR_INVALID with nothing written; size 2^a is verified (identity points: a verdict,
    not an error).  In a child process with a timeout, so that a verifier that forms Z_D over such a size fails the test
    instead of hanging it."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    cases = [[0, 2], [3, 9], [28, (1 << 28) + 1], [3, 1 << 63], [28, 1 << 63], [0, 1], [3, 8], [10, 1 << 10]]
    env = dict(os.environ, PYTHONPATH=root)
    try:
        run = subprocess.run([sys.executable, "-c", _PROBE, os.path.join(root, "tests", "golden", "srs_g2.bin"),
                              json.dumps(cases)], capture_output=True, text=True, timeout=60, env=env, cwd=root)
    except subprocess.TimeoutExpired as exc:
        pytest.fail(f"the host link verifier did not return within 60 s: {exc.stdout!r}")
    assert run.returncode == 0, run.stderr
    got = json.loads(run.stdout.strip().splitlines()[-1])
    refused = [[_lib.B200_ERR_INVALID, 7]] * 5
    assert got[:5] == refused, got
    assert [rc for rc, _ in got[5:]] == [_lib.B200_OK] * 3 and all(v in (0, 1) for _, v in got[5:]), got
