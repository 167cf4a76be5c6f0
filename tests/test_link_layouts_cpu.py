"""The link-proof inputs of `link_layouts.py` (which `test_gpu_link_layouts.py` gives the device) checked against the oracle
alone: every case has the shape it claims (N, q_len, the wrap, len = N, ...); the oracle links every constructed pair
(rc 0) and its link verifier accepts the proof; a pair that differs on exactly one root of the group is refused (rc 2);
and a layout shifted by one no longer verifies, except where the shift keeps the group's roots (the whole subgroup) or
the two polynomials are equal."""
import numpy as np
import pytest

import link_layouts as ll

TAU = 0x1D2C3B4A59687706F5E4D3C2B1A09F8E7D6C5B4A39281706F5E4D3C2B1A0987  # conftest's SRS_2_16_TAU
NAMES = [c.name for c in ll.CASES]


@pytest.fixture(scope="module")
def env(oracle):
    class E:
        pass
    e = E()
    e.tau = oracle.int_to_limbs(TAU % ll.R * ll.MONT % ll.R)
    e.srs = oracle.srs_from_tau(e.tau, max(c.len for c in ll.CASES))
    return e


def commit(oracle, srs, vals):
    xy, inf = oracle.msm(srs[:len(vals)], oracle.ints_to_array(vals))
    return np.zeros(8, dtype=np.uint64) if inf else xy


@pytest.mark.parametrize("name", NAMES)
def test_case_has_the_shape_it_claims(oracle, name):
    c = ll.BY_NAME[name]
    assert ll.domain_n(c.len) == c.N and c.len - c.size == c.q_len
    assert 1 <= c.size < c.len and c.size <= 1 << c.alignment
    rts = ll.roots(oracle, c)
    assert len(set(rts)) == c.size
    g = ll.generator(oracle, c.alignment)
    assert pow(g, 1 << c.alignment, ll.R) == 1 and (c.alignment == 0 or pow(g, 1 << (c.alignment - 1), ll.R) != 1)
    assert c.wraps == (name in ("wraps", "whole_group_shifted"))
    assert (1 in rts) == (c.wraps or c.offset % (1 << c.alignment) == 0)
    same = ll.roots(oracle, ll.Case("", c.alignment, c.offset % (1 << c.alignment), c.size, c.len1, c.len2, c.N, c.q_len))
    assert rts == same  # an offset names its roots modulo 2^alignment
    assert c.identical == (name == "identical")
    log_n = c.N.bit_length() - 1
    claims = {
        "size_one": c.size == 1,
        "q_len_one": c.q_len == 1,
        "whole_group": c.offset == 0 and c.size == 1 << c.alignment
                       and ll.vanishing(rts) == [ll.R - 1] + [0] * (c.size - 1) + [1],
        "wraps": c.offset < 1 << c.alignment < c.offset + c.size,
        "wide_alignment": c.alignment > log_n,
        "no_slack": c.len == c.N,
        "len1_lt_len2": c.len1 < c.len2,
        "len1_far_above_len2": c.len1 > 32 * c.len2,
        "len1_just_above_len2": c.len1 == c.len2 + 1 == c.N // 2 + 1,
        "identical": c.len1 == c.len2,
        "largest_srs": c.len == (1 << 17) + 2 and c.N == 1 << 18,
        "offset_past_group": c.offset == (1 << c.alignment) + 3,
        "offset_2_63": c.offset == (1 << 63) + 5 and c.offset < 1 << 64,
        "whole_group_shifted": c.offset == 5 and c.size == 1 << c.alignment
                               and ll.vanishing(rts) == [ll.R - 1] + [0] * (c.size - 1) + [1],
        "alignment_zero": c.alignment == 0 and c.size == 1 and rts == [1],
        "alignment_28": c.alignment == 28 and c.N == 32,
    }
    assert claims[name]


@pytest.mark.parametrize("name", NAMES)
def test_oracle_links_the_constructed_pair(oracle, env, name):
    c = ll.BY_NAME[name]
    a1, a2 = ll.pair(oracle, c, seed=0x11 + NAMES.index(name))
    d = ll.poly_add(a1, a2, -1)
    assert all(ll.poly_eval(d, r) == 0 for r in ll.roots(oracle, c))
    m1, m2 = ll.to_mont(a1), ll.to_mont(a2)
    c1, c2 = commit(oracle, env.srs, a1), commit(oracle, env.srs, a2)
    rc, lp, eta = oracle.plonk_link(m1, m2, c1, c2, c.alignment, c.offset, c.size, env.srs)
    assert rc == 0
    arr = np.frombuffer(bytes(lp), dtype=np.uint64)
    assert (not arr.any()) == c.identical  # equal polynomials: identity quotient and opening
    assert oracle.plonk_link_verify_known_tau(c1, c2, c.alignment, c.offset, c.size, lp, env.tau)
    # one row further: other roots, unless the group is the whole subgroup (same roots) or the difference is zero
    keeps = c.identical or c.size == 1 << c.alignment
    assert oracle.plonk_link_verify_known_tau(c1, c2, c.alignment, c.offset + 1, c.size, lp, env.tau) == keeps


@pytest.mark.parametrize("j", ["first", "middle", "last"])
def test_oracle_refuses_a_one_root_mismatch(oracle, env, j):
    c = ll.BY_NAME["wraps"]
    idx = {"first": 0, "middle": c.size // 2, "last": c.size - 1}[j]
    a1, a2 = ll.pair(oracle, c, seed=77)
    bad = ll.mismatch(oracle, c, a1, idx, 0xC0FFEE)
    assert len(bad) == c.len1
    d = ll.poly_add(bad, a2, -1)
    assert [ll.poly_eval(d, r) != 0 for r in ll.roots(oracle, c)] == [i == idx for i in range(c.size)]
    rc, _, _ = oracle.plonk_link(ll.to_mont(bad), ll.to_mont(a2), np.zeros(8, np.uint64), np.zeros(8, np.uint64),
                                 c.alignment, c.offset, c.size, env.srs)
    assert rc == 2
