"""Poseidon2 batch hashing (SURVEY §8(f) f4).  CPU: the oracle restatement of
crates/crypto/src/hash/poseidon2.rs reproduces the published known answer with the reference's
constants.  GPU: the device kernels match the oracle bit-exactly."""
import json
import os

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIX = os.path.join(ROOT, "tests", "golden", "poseidon2.json")


def test_oracle_matches_published_kat(pyoracle):
    py = pyoracle
    full, partial = py.poseidon2_load_constants(FIX)
    assert len(full) == 24 and len(partial) == 56
    kat = json.load(open(FIX))["kat_permutation_0_1_2"]["output"]
    assert py.poseidon2_permute([0, 1, 2], full, partial) == [int(v, 16) for v in kat]


def test_generated_header_matches_fixture(pyoracle):
    """The constants compiled into the product are the reference's (Montgomery form of the fixture)."""
    import re
    py = pyoracle
    full, partial = py.poseidon2_load_constants(FIX)
    txt = open(os.path.join(ROOT, "renegade_b200", "csrc", "poseidon2_constants.h")).read()
    rows = re.findall(r"\{((?:0x[0-9a-f]{8}u(?:, )?){8})\}", txt)
    vals = [sum(int(w.rstrip("u"), 16) << (32 * i) for i, w in enumerate(r.split(", "))) for r in rows]
    assert vals == [py.to_mont(v, py.R) for v in full + partial]


@pytest.mark.gpu
def test_gpu_permutation_and_hash(ctx, oracle, pyoracle):
    """The published known answer through the device permutation; then every output of 300 random permutations and of
    130 sponge hashes per length 0..7 against the C oracle (itself pinned by tests/test_poseidon2_oracle_cpu.py)."""
    from renegade_b200.backend import compute_poseidon_hash_batch, poseidon2_permute_batch
    py = pyoracle
    to_m = lambda vals: oracle.ints_to_array([py.to_mont(v, py.R) for v in vals])
    from_m = lambda arr: [py.from_mont(v, py.R) for v in oracle.array_to_ints(arr)]
    # the published known answer through the device permutation
    kat = [int(v, 16) for v in json.load(open(FIX))["kat_permutation_0_1_2"]["output"]]
    st = to_m([0, 1, 2]).reshape(1, 3, 4)
    assert from_m(poseidon2_permute_batch(ctx, st).reshape(3, 4)) == kat
    # random states
    import random
    rnd = random.Random(5)
    states = to_m([rnd.randrange(py.R) for _ in range(3 * 300)]).reshape(-1, 3, 4)
    assert np.array_equal(poseidon2_permute_batch(ctx, states), oracle.poseidon2_permute_batch(states))
    # sponge hashes of every length 0..7 (odd lengths leave the rate half full; 0 = hash of nothing)
    for ln in range(0, 8):
        arr = to_m([rnd.randrange(py.R) for _ in range(130 * ln)]).reshape(130, ln, 4)
        assert np.array_equal(compute_poseidon_hash_batch(ctx, arr), oracle.poseidon2_hash_batch(arr)), ln


@pytest.mark.gpu
def test_gpu_merkle_roots_and_csprng_streams(ctx, oracle, pyoracle):
    """The batch callers of the witness side (SURVEY §8(f) f4): Merkle roots of openings of height 10 (`MERKLE_HEIGHT`,
    constants/src/lib.rs:50) and Poseidon CSPRNG stream values H(seed, i) (darkpool-types/src/csprng.rs:30-75), every
    output against the C oracle's Poseidon2 (one batched two-to-one hash per level, H(seed, first + j))."""
    import random
    from renegade_b200.backend import csprng_batch, merkle_root_batch
    py = pyoracle
    to_m = lambda vals: oracle.ints_to_array([py.to_mont(v, py.R) for v in vals])
    rnd = random.Random(11)
    batch, height = 67, 10
    leaves = to_m([rnd.randrange(py.R) for _ in range(batch)])
    sisters = to_m([rnd.randrange(py.R) for _ in range(batch * height)]).reshape(batch, height, 4)
    bits = np.array([[rnd.random() < 0.5 for _ in range(height)] for _ in range(batch)], dtype=np.uint8)
    got = merkle_root_batch(ctx, leaves, sisters, bits)
    assert np.array_equal(got, oracle.poseidon2_merkle_roots(leaves, sisters, bits))
    # height 0: the root is the leaf hash itself
    assert np.array_equal(merkle_root_batch(ctx, leaves[:3], np.zeros((3, 0, 4), dtype=np.uint64),
                                            np.zeros((3, 0), dtype=np.uint8)), leaves[:3])
    seeds = to_m([rnd.randrange(py.R) for _ in range(9)])
    first = [rnd.randrange(0, 1 << 40) for _ in range(9)]
    assert np.array_equal(csprng_batch(ctx, seeds, first, 5), oracle.poseidon2_csprng(seeds, first, 5))
