"""CPU: the C Poseidon2 oracle (oracle/poseidon2_oracle.c) that the GPU Poseidon2 tests compare every output with is
pinned here before any of them relies on it — the published known answer, the pure-Python restatement
(bn254_py.poseidon2_permute / poseidon2_hash) on edge, round-targeted and seeded random states and on sponges of many
lengths, and the Merkle-root and CSPRNG compositions against their Python definitions.  The edge-state builders of
tests/poseidon2_shapes.py are checked against their own claims."""
import json
import time

import numpy as np
import pytest

import poseidon2_shapes as P2


@pytest.fixture(scope="module")
def rc(pyoracle, oracle):
    return pyoracle.poseidon2_load_constants(oracle.POSEIDON2_FIXTURE)


def mont_array(oracle, pyoracle, vals):
    return oracle.ints_to_array([pyoracle.to_mont(v, pyoracle.R) for v in vals])


def plain(oracle, pyoracle, arr):
    return [pyoracle.from_mont(v, pyoracle.R) for v in oracle.array_to_ints(arr)]


def test_c_oracle_reproduces_the_published_kat(oracle, pyoracle):
    kat = [int(v, 16) for v in json.load(open(oracle.POSEIDON2_FIXTURE))["kat_permutation_0_1_2"]["output"]]
    got = oracle.poseidon2_permute_batch(mont_array(oracle, pyoracle, [0, 1, 2]).reshape(1, 3, 4))
    assert plain(oracle, pyoracle, got) == kat


def test_targeted_states_reach_their_targets(pyoracle, rc):
    """Each round-targeted state, run forward with a hook, presents its target residue to the S-box of its round and
    lane; the hooked forward permutation is bn254_py's."""
    full, partial = rc
    cases = P2.targeted_states(full, partial)
    assert len(cases) == len(P2.POSITIONS) * len(P2.TARGETS) == 27 * 7
    for rd, lane, t, st in cases:
        x = [P2.unmont(v) for v in st]
        out, seen = P2.forward_sbox_inputs(x, full, partial)
        assert len(seen) == 8 * 3 + 56
        assert P2.mont(seen[(rd, lane)]) == t, (rd, lane, t)
        assert out == pyoracle.poseidon2_permute(x, full, partial)


def test_edge_states_are_what_they_claim(pyoracle):
    R = pyoracle.R
    states = P2.edge_states()
    ops = P2.operands(R)
    assert len(states) == 4 * len(ops) + 3 * 2 * 4
    assert {0, 1, R - 1, (R - 1) // 2, (R + 1) // 2, P2.MONT % R, 1 << 253} <= set(ops)
    assert ("all=%#x" % (R - 1), [R - 1] * 3) in states and 3 * (R - 1) >= 2 * R  # the MDS sum wraps twice
    mds0 = [(lab, s) for lab, s in states if lab.startswith("mds0")]
    assert len(mds0) == 24
    for lab, s in mds0:
        lane, t = int(lab[5]), int(lab.split("=")[1], 16)
        assert P2.external_mds(s)[lane] == t and all(0 <= v < R for v in s)


def test_c_permutation_equals_python(oracle, pyoracle, rc):
    """Edge states, round-targeted states and 2000 seeded random states: every output equals the Python restatement."""
    full, partial = rc
    residues = [s for _, s in P2.edge_states()] + [s for *_, s in P2.targeted_states(full, partial)]
    arr = np.concatenate([oracle.ints_to_array([v for s in residues for v in s]),
                          oracle.splitmix_fr(0x9E02, 3 * 2000, montgomery=True)]).reshape(-1, 3, 4)
    got = oracle.poseidon2_permute_batch(arr)
    inp, out = plain(oracle, pyoracle, arr), plain(oracle, pyoracle, got)
    bad = [i for i in range(arr.shape[0]) if out[3 * i:3 * i + 3] != pyoracle.poseidon2_permute(inp[3 * i:3 * i + 3], full, partial)]
    assert not bad, f"{len(bad)} of {arr.shape[0]} states differ, first {bad[:5]}"


@pytest.mark.parametrize("ln", list(range(34)) + [257, 1000])
def test_c_sponge_equals_python(oracle, pyoracle, rc, ln):
    full, partial = rc
    rows = 3 if ln < 34 else 1
    vals = oracle.splitmix_fr(0x5B0 + ln, rows * ln, montgomery=True).reshape(rows, ln, 4)
    if ln >= 2:  # edge operands in the absorbed values too: r - 1 twice (the rate lanes wrap), then 0
        vals[0, :2] = oracle.ints_to_array([pyoracle.R - 1] * 2)
        vals[-1, -1] = 0
    got = plain(oracle, pyoracle, oracle.poseidon2_hash_batch(vals))
    for i in range(rows):
        assert got[i] == pyoracle.poseidon2_hash(plain(oracle, pyoracle, vals[i]), full, partial), (ln, i)


def test_merkle_and_csprng_compositions_equal_their_definitions(oracle, pyoracle, rc):
    full, partial = rc
    H = lambda a, b: pyoracle.poseidon2_hash([a, b], full, partial)
    rng = np.random.default_rng(0x3E)
    for batch, height in ((1, 0), (3, 1), (4, 3), (2, 10)):
        leaves = oracle.splitmix_fr(0x1EAF + height, batch, montgomery=True)
        sis = oracle.splitmix_fr(0x5155 + height, batch * height, montgomery=True).reshape(batch, height, 4)
        bits = rng.choice(np.array([0, 1, 2, 255], dtype=np.uint8), size=(batch, height))
        got = plain(oracle, pyoracle, oracle.poseidon2_merkle_roots(leaves, sis, bits))
        for i in range(batch):
            cur = plain(oracle, pyoracle, leaves[i])[0]
            for lvl, s in enumerate(plain(oracle, pyoracle, sis[i])):
                cur = H(s, cur) if bits[i, lvl] else H(cur, s)
            assert got[i] == cur, (batch, height, i)
    # CSPRNG: H(seed, first + j) with the index a plain integer; streams across 2^32 (the low 32-bit limb carries) and
    # up to the last u64 index
    seeds = oracle.splitmix_fr(0xC5, 3, montgomery=True)
    first = [(1 << 32) - 3, 0, (1 << 64) - 6]
    got = oracle.poseidon2_csprng(seeds, first, 6)
    for s in range(3):
        seed = plain(oracle, pyoracle, seeds[s])[0]
        assert plain(oracle, pyoracle, got[s]) == [H(seed, first[s] + j) for j in range(6)], s
    assert H(plain(oracle, pyoracle, seeds[0])[0], 1 << 32) == plain(oracle, pyoracle, got[0, 3])[0]


def test_oracle_time_per_permutation(oracle, capsys):
    """Reports the C oracle's cost (not a bound): one thread, then all of this host's threads."""
    arr = oracle.splitmix_fr(0x7173, 3 * (1 << 14), montgomery=True).reshape(-1, 3, 4)
    threads = oracle.num_threads()
    res = {}
    try:
        for k in (1, threads):
            oracle.set_num_threads(k)
            t = time.perf_counter()
            oracle.poseidon2_permute_batch(arr)
            res[k] = (time.perf_counter() - t) / arr.shape[0] * 1e6
    finally:
        oracle.set_num_threads(threads)
    with capsys.disabled():
        print(f"\nC Poseidon2 oracle: {res[1]:.2f} us per permutation on one thread, {res[threads]:.2f} us "
              f"wall per permutation on {threads} threads")
