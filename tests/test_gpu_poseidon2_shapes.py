"""GPU: the four Poseidon2 batch calls (`b200_poseidon2_{permute,hash,merkle_root,csprng}_batch`) at the shapes and
values where a one-thread-per-hash kernel goes wrong, EVERY output of every call compared with the C oracle
(oracle/poseidon2_oracle.c, pinned by tests/test_poseidon2_oracle_cpu.py) with np.array_equal:

- permutations of the edge and round-targeted states of tests/poseidon2_shapes.py, and of seeded batches across the
  128-thread block boundaries up to 2^20 states; in place on device, pageable, pinned and managed memory;
- sponges of every length 0 ... 33 and of 257, 1000 and 4097 scalars, 2^20 two-to-one hashes on device buffers, an
  empty sponge with no input pointer;
- Merkle roots of heights 0 ... 64 with every `is_right` pattern (bytes 2 and 255 are right), a sister equal to the
  running hash; height 65 refused;
- CSPRNG streams whose index carries out of its low 32-bit limb, up to the last u64 index, across block boundaries;
- argument errors, empty batches, the prover's workspace (`plonk_ws`) these calls grow between replayed proofs, and
  first calls in fresh processes (one context, and two contexts racing from two threads)."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

import poseidon2_shapes as P2
from renegade_b200 import _lib
from renegade_b200.backend import compute_poseidon_hash_batch, csprng_batch, merkle_root_batch, poseidon2_permute_batch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def same(got, exp, what):
    got, exp = np.asarray(got, dtype=np.uint64), np.asarray(exp, dtype=np.uint64)
    assert got.shape == exp.shape, (what, got.shape, exp.shape)
    if not np.array_equal(got, exp):
        bad = np.nonzero((got.reshape(got.shape[0], -1) != exp.reshape(exp.shape[0], -1)).any(axis=1))[0]
        pytest.fail(f"{what}: {len(bad)} of {got.shape[0]} outputs differ from the oracle, first at {bad[:8].tolist()}")


def rand_fr(oracle, seed, n):
    return oracle.splitmix_fr(seed, n, montgomery=True)


# ---- permute ---------------------------------------------------------------------------------------------------------
def test_permute_edge_and_round_targeted_states(ctx, oracle, pyoracle):
    full, partial = pyoracle.poseidon2_load_constants(oracle.POSEIDON2_FIXTURE)
    states = [s for _, s in P2.edge_states()] + [s for *_, s in P2.targeted_states(full, partial)]
    arr = oracle.ints_to_array([v for s in states for v in s]).reshape(-1, 3, 4)
    same(poseidon2_permute_batch(ctx, arr), oracle.poseidon2_permute_batch(arr), "edge states")


@pytest.mark.parametrize("batch", [1, 127, 128, 129, 255, 256, 257, 65537, 1 << 20])
def test_permute_random_batches(ctx, oracle, batch):
    arr = rand_fr(oracle, 0x9E0 + batch, 3 * batch).reshape(batch, 3, 4)
    same(poseidon2_permute_batch(ctx, arr), oracle.poseidon2_permute_batch(arr), f"batch {batch}")


@pytest.fixture(scope="module")
def sources():
    from test_gpu_witness_shapes import Sources
    s = Sources()
    yield s
    s.close()


@pytest.mark.parametrize("kind", ["numpy", "pinned", "device", "device+16", "device+8", "managed"])
def test_permute_in_place_on_every_pointer_kind(ctx, oracle, sources, kind):
    """The states are permuted where they are: read back from the caller's own buffer."""
    arr = rand_fr(oracle, 0xB1D, 3 * 4099).reshape(-1, 3, 4)
    p = sources.pointer(arr.copy(), kind)
    ptr = p.ctypes.data_as(C.c_void_p) if kind == "numpy" else C.c_void_p(p)
    _lib.check(ctx._lib.b200_poseidon2_permute_batch(ctx._h, ptr, arr.shape[0]))
    got = np.zeros_like(arr)
    assert sources._rt.cudaMemcpy(got.ctypes.data_as(C.c_void_p), ptr, C.c_size_t(arr.nbytes), 4) == 0  # Default
    same(got, oracle.poseidon2_permute_batch(arr), kind)


# ---- hash ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("ln", range(34))
def test_hash_every_length_up_to_33(ctx, oracle, ln):
    """Both parities (an odd length squeezes with the rate half full) on batches of 1, 128 and 129; row 0 of each batch
    absorbs r - 1 everywhere, row 1 zeros."""
    for batch in (1, 128, 129):
        vals = rand_fr(oracle, (ln << 8) + batch, batch * ln).reshape(batch, ln, 4)
        vals[0] = oracle.ints_to_array([P2.R - 1] * ln).reshape(ln, 4)
        if batch > 1:
            vals[1] = 0
        same(compute_poseidon_hash_batch(ctx, vals), oracle.poseidon2_hash_batch(vals), f"len {ln} batch {batch}")


@pytest.mark.parametrize("ln,batch", [(257, 5), (1000, 3), (4097, 3)])
def test_hash_long_sponges(ctx, oracle, ln, batch):
    vals = rand_fr(oracle, 0x10E6 + ln, batch * ln).reshape(batch, ln, 4)
    same(compute_poseidon_hash_batch(ctx, vals), oracle.poseidon2_hash_batch(vals), f"len {ln}")


def test_hash_2_20_two_to_one_on_device_buffers(ctx, oracle):
    """tools/poseidon_bench.py's workload: inputs made on the device by b200_splitmix_fr_device, device in, device out."""
    import torch
    batch = 1 << 20
    d_in = torch.empty((batch, 2, 4), dtype=torch.int64, device="cuda")
    d_out = torch.empty((batch, 4), dtype=torch.int64, device="cuda")
    torch.cuda.synchronize()
    ctx.splitmix_fr_device(0x90, batch * 2, d_in.data_ptr(), montgomery=True)
    _lib.check(ctx._lib.b200_poseidon2_hash_batch(ctx._h, C.c_void_p(d_in.data_ptr()), batch, 2, C.c_void_p(d_out.data_ptr())))
    vals = rand_fr(oracle, 0x90, 2 * batch).reshape(batch, 2, 4)
    same(d_in.cpu().numpy().view(np.uint64), vals, "device inputs")
    same(d_out.cpu().numpy().view(np.uint64), oracle.poseidon2_hash_batch(vals), "2^20 hashes")


def test_hash_of_nothing_with_no_input_pointer(ctx, oracle):
    out = np.zeros((5, 4), dtype=np.uint64)
    _lib.check(ctx._lib.b200_poseidon2_hash_batch(ctx._h, None, 5, 0, out.ctypes.data_as(C.c_void_p)))
    same(out, oracle.poseidon2_hash_batch(np.zeros((5, 0, 4), dtype=np.uint64)), "len 0")


# ---- Merkle roots ----------------------------------------------------------------------------------------------------
def merkle_case(oracle, batch, height, seed):
    """Leaves, sisters and is_right bytes; rows cycle through is_right all 0, all 1, alternating, random 0 / 1 and random
    bytes from {0, 1, 2, 255}; every 7th row's sister at level min(height - 1, 5) is the running hash there."""
    rng = np.random.default_rng(seed)
    leaves = rand_fr(oracle, seed, batch)
    sis = rand_fr(oracle, seed + 1, batch * height).reshape(batch, height, 4)
    bits = np.zeros((batch, height), dtype=np.uint8)
    for i in range(batch):
        bits[i] = [np.zeros(height), np.ones(height), np.arange(height) % 2, rng.integers(0, 2, height),
                   rng.choice([0, 1, 2, 255], height)][i % 5]
    if height:
        lvl = min(height - 1, 5)
        rows = np.arange(0, batch, 7)
        sis[rows, lvl] = oracle.poseidon2_merkle_roots(leaves[rows], sis[rows, :lvl], bits[rows, :lvl])
    return leaves, sis, bits


MERKLE = [(h, 129) for h in (0, 1, 2, 10, 32, 63, 64)] + [(0, 1), (64, 1), (0, 4097), (10, 4097), (64, 4097)]


@pytest.mark.parametrize("height,batch", MERKLE)
def test_merkle_roots(ctx, oracle, height, batch):
    leaves, sis, bits = merkle_case(oracle, batch, height, seed=(height << 16) + batch)
    if batch >= 129 and height:
        assert {2, 255} <= set(bits[4::5].ravel().tolist())  # the header's `!= 0`: these bytes count as right
    same(merkle_root_batch(ctx, leaves, sis, bits), oracle.poseidon2_merkle_roots(leaves, sis, bits),
         f"height {height} batch {batch}")


def test_merkle_height_limits(ctx, oracle):
    leaves = rand_fr(oracle, 0x65, 3)
    out = np.zeros((3, 4), dtype=np.uint64)
    sis = rand_fr(oracle, 0x66, 3 * 65)
    bits = np.ones(3 * 65, dtype=np.uint8)
    P = lambda a: a.ctypes.data_as(C.c_void_p)
    assert ctx._lib.b200_poseidon2_merkle_root_batch(ctx._h, P(leaves), P(sis), P(bits), 3, 65, P(out)) == _lib.B200_ERR_INVALID
    assert not out.any()
    _lib.check(ctx._lib.b200_poseidon2_merkle_root_batch(ctx._h, P(leaves), None, None, 3, 0, P(out)))
    same(out, leaves, "height 0 with no sisters")


# ---- CSPRNG ----------------------------------------------------------------------------------------------------------
FIRSTS = [0, (1 << 32) - 3, 1 << 40, 1 << 63]


@pytest.mark.parametrize("count", [1, 2, 3, 127, 128, 129, 1000])
def test_csprng_index_edges(ctx, oracle, count):
    """One stream per first index, the last one ending on index 2^64 - 1; with 2^32 - 3 the stream crosses into the
    second 32-bit limb of the index (for count >= 4)."""
    first = FIRSTS + [(1 << 64) - count]
    seeds = rand_fr(oracle, 0xC0 + count, len(first))
    same(csprng_batch(ctx, seeds, first, count), oracle.poseidon2_csprng(seeds, first, count), f"count {count}")


def test_csprng_many_streams_with_edge_seeds(ctx, oracle):
    seeds = oracle.ints_to_array(P2.operands(P2.R))
    rng = np.random.default_rng(0xC5)
    first = [int(rng.choice(FIRSTS)) + int(rng.integers(0, 1 << 20)) for _ in range(seeds.shape[0])]
    same(csprng_batch(ctx, seeds, first, 5), oracle.poseidon2_csprng(seeds, first, 5), "edge seeds")


# ---- argument errors -------------------------------------------------------------------------------------------------
def test_argument_errors_and_empty_batches(ctx, oracle):
    L, h = ctx._lib, ctx._h
    P = lambda a: a.ctypes.data_as(C.c_void_p)
    st = rand_fr(oracle, 0xA1, 6)
    idx = np.zeros(2, dtype=np.uint64)
    bits = np.zeros(2, dtype=np.uint8)
    out = np.full((2, 4), 0xABABABABABABABAB, dtype=np.uint64)
    keep = out.copy()
    INV = _lib.B200_ERR_INVALID
    # a null context, and a null output, for all four calls
    assert L.b200_poseidon2_permute_batch(None, P(st), 2) == INV
    assert L.b200_poseidon2_hash_batch(None, P(st), 2, 1, P(out)) == INV
    assert L.b200_poseidon2_merkle_root_batch(None, P(st), P(st), P(bits), 2, 1, P(out)) == INV
    assert L.b200_poseidon2_csprng_batch(None, P(st), P(idx), 2, 1, P(out)) == INV
    assert L.b200_poseidon2_permute_batch(h, None, 2) == INV
    assert L.b200_poseidon2_hash_batch(h, P(st), 2, 1, None) == INV
    assert L.b200_poseidon2_merkle_root_batch(h, P(st), P(st), P(bits), 2, 1, None) == INV
    assert L.b200_poseidon2_csprng_batch(h, P(st), P(idx), 2, 1, None) == INV
    # batch 0 (and count 0) is OK and writes nothing
    st0 = st.copy()
    assert L.b200_poseidon2_permute_batch(h, P(st), 0) == _lib.B200_OK
    assert L.b200_poseidon2_hash_batch(h, P(st), 0, 3, P(out)) == _lib.B200_OK
    assert L.b200_poseidon2_merkle_root_batch(h, P(st), P(st), P(bits), 0, 1, P(out)) == _lib.B200_OK
    assert L.b200_poseidon2_csprng_batch(h, P(st), P(idx), 0, 4, P(out)) == _lib.B200_OK
    assert L.b200_poseidon2_csprng_batch(h, P(st), P(idx), 2, 0, P(out)) == _lib.B200_OK
    assert np.array_equal(out, keep) and np.array_equal(st, st0)


# ---- the prover's workspace ------------------------------------------------------------------------------------------
def test_calls_between_replayed_proofs(oracle, pyoracle):
    """The four calls stage their data in `plonk_ws`, the workspace the single-proof CUDA graphs capture.  On a context
    of its own, whose workspace only a 2^7 proof has sized (well under 1 MiB), a batch of 2^20 two-to-one hashes needs
    96 MiB: the buffer is freed and allocated again between replayed proofs of one key.  The graphs captured on the old
    buffer must not be replayed (csrc/plonk.cu buffer_fingerprint).  The wires are staged into the workspace outside the
    graphs, so the proof right after the move uses a witness B the earlier proofs did not: a graph still reading the
    freed buffer would see witness A's wires there, and its bytes would not equal the oracle's proof of B.  The graph
    count (7 submissions a proof) is the same for a capture and a replay: it only shows that the graph path ran.  A
    small call between two replayed proofs leaves both proofs and its own outputs right."""
    import renegade_b200 as rb
    import witness_shapes as ws
    from test_gpu_graphs import SEGMENTS, check, make
    c = rb.Context(0)  # the session context's workspace is already larger than the batch below
    try:
        c.use_graphs(True)
        log_n = 7
        circ, srs, bases, pk, opk = make(c, oracle, pyoracle, log_n, seed=0x9052)
        a, b = (ws.with_witness(circ, w) for w in ws.dense_witnesses(circ, 2, seed=0x9052))
        check(c, oracle, log_n, a, srs, pk, opk, 1)  # eager
        check(c, oracle, log_n, a, srs, pk, opk, 2)  # captured
        vals = rand_fr(oracle, 0x6E0, 1 << 21).reshape(-1, 2, 4)
        same(compute_poseidon_hash_batch(c, vals), oracle.poseidon2_hash_batch(vals), "growing hash batch")
        g0 = c.graph_launches()
        check(c, oracle, log_n, b, srs, pk, opk, 3)  # captured again on the new workspace
        check(c, oracle, log_n, a, srs, pk, opk, 4)  # replayed
        small = rand_fr(oracle, 0x6E1, 3 * 5).reshape(5, 3, 4)
        same(poseidon2_permute_batch(c, small), oracle.poseidon2_permute_batch(small), "small permute between proofs")
        seeds = rand_fr(oracle, 0x6E2, 2)
        same(csprng_batch(c, seeds, [7, (1 << 32) - 1], 3), oracle.poseidon2_csprng(seeds, [7, (1 << 32) - 1], 3),
             "small csprng between proofs")
        check(c, oracle, log_n, b, srs, pk, opk, 5)  # replayed
        assert c.graph_launches() - g0 == 3 * SEGMENTS
        pk.free()
        bases.free()
    finally:
        c.close()


# ---- first calls -----------------------------------------------------------------------------------------------------
FIRST_CALL = r"""
import sys, threading
import numpy as np
sys.path.insert(0, sys.argv[1])
import renegade_b200 as rb
from renegade_b200.backend import poseidon2_permute_batch
inp = np.load(sys.argv[2])
states = [inp[k] for k in sorted(inp.files)]
ctxs = [rb.Context(0) for _ in states]  # no Poseidon2 work on the device before the calls below
out = [None] * len(states)
go = threading.Barrier(len(states))
def run(i):
    go.wait()
    out[i] = poseidon2_permute_batch(ctxs[i], states[i])
threads = [threading.Thread(target=run, args=(i,)) for i in range(len(states))]
for t in threads:
    t.start()
for t in threads:
    t.join()
np.savez(sys.argv[3], *out)
"""


@pytest.mark.parametrize("contexts,batch", [(1, 1 << 16), (2, 1 << 14)])
def test_first_calls_in_a_fresh_process(oracle, tmp_path, contexts, batch):
    """The first Poseidon2 call of a process uploads the round constants (once per device): one context whose first
    GPU work is a 2^16-state permutation, and two contexts on device 0 making their first calls from two threads at
    once (one uploads, the other waits for it).  Run once each."""
    states = [rand_fr(oracle, 0xF1 + i, 3 * batch).reshape(batch, 3, 4) for i in range(contexts)]
    np.savez(tmp_path / "in.npz", *states)
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", FIRST_CALL, ROOT,
                                                                           str(tmp_path / "in.npz"), str(tmp_path / "out.npz")]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-3000:]
    got = np.load(tmp_path / "out.npz")
    for i in range(contexts):
        same(got[f"arr_{i}"], oracle.poseidon2_permute_batch(states[i]), f"context {i}")


def test_context_on_a_second_device(oracle):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs a 2-GPU box")
    import renegade_b200 as rb
    c1 = rb.Context(1)
    try:
        arr = rand_fr(oracle, 0xD1, 3 * 1000).reshape(-1, 3, 4)
        same(poseidon2_permute_batch(c1, arr), oracle.poseidon2_permute_batch(arr), "device 1")
        vals = rand_fr(oracle, 0xD2, 129 * 9).reshape(129, 9, 4)
        same(compute_poseidon_hash_batch(c1, vals), oracle.poseidon2_hash_batch(vals), "device 1 hash")
    finally:
        c1.close()
