"""The device wiring (`wiring.cu`) and the witness-vector prover at the shapes of tests/witness_shapes.py: full size
(2^16, 2^17), both sides of each digit of the sort up to a 32-bit index, every witness pointer kind, batches past one gather group of
`k_gather_wires`, staging that outgrows the NTT scratch under replayed graphs, and the public-input extremes through
all three verifiers.

References: `wpk` is the key `b200_plonk_preprocess_wiring` makes, `pk` the key `b200_plonk_preprocess` makes from
test_prove_witness_cpu.wiring_permutation; a witness proof must equal the table proof of the expanded table byte for
byte, and the oracle checks both where it is affordable.  No proof is asked of a key whose indices lie past a real
witness buffer."""
import ctypes as C

import numpy as np
import pytest

import witness_shapes as ws
from renegade_b200 import _lib, synth
from renegade_b200.backend import PlonkKzgSnark, VerifyingKey
from test_gpu_prove_witness import TAU, from_table, from_witness, keys, unsatisfying
from test_prove_witness_cpu import expand, wiring_permutation

pytestmark = pytest.mark.gpu

INVALID, UNSAT = -1, -7
LOG_MAX = 17


@pytest.fixture(scope="module")
def tau(oracle, pyoracle):
    return oracle.int_to_limbs(pyoracle.to_mont(TAU % pyoracle.R, pyoracle.R))


@pytest.fixture(scope="module")
def srs(oracle, tau):
    """2^17 + 3 powers of conftest's SRS_2_16_TAU (srs_2_16_g2 is its G2 pair); a domain of n takes the first n + 3."""
    return oracle.srs_from_tau(tau, (1 << LOG_MAX) + 3)


def equal_keys(ctx, bases, circ, num_vars=None):
    """keys(), asserted equal: selector and sigma commitments, and the key from the wiring holds num_vars"""
    wpk, pk = keys(ctx, bases, circ, num_vars)
    assert (wpk.selector_comms == pk.selector_comms).all()
    assert (wpk.sigma_comms == pk.sigma_comms).all()
    assert wpk.num_vars == (circ.num_vars if num_vars is None else num_vars)
    return wpk, pk


def same_proofs(ctx, wpk, pk, circ, seed):
    """prove_witness = prove_with_link_hint of the expanded table: proof, link polynomial, challenges; public inputs.
    Returns (the proof, its blinders)."""
    bl = synth.splitmix_blinders(seed)
    proof, hint, pub, ch = PlonkKzgSnark.prove_witness(ctx, wpk, circ.witness, bl, want_challenges=True)
    assert (bytes(proof), hint.linking_wire_poly.tobytes(), ch.tobytes()) == from_table(ctx, pk, circ, bl)
    assert (pub == circ.witness[circ.wire_vars[4, :circ.num_inputs]]).all()
    return proof, bl


def free(*objs):
    for o in objs:
        o.free()


# ---- keys and proofs on both sides of each sort digit ---------------------------------------------------------------------------
@pytest.mark.parametrize("num_vars", ws.INDEX_WIDTHS)
def test_index_width_keys_and_proofs(ctx, srs, num_vars):
    s = ws.index_width(num_vars)
    circ = s.circ
    assert int(circ.wire_vars.max()) == num_vars - 1 and f"end_bit {ws.end_bit(num_vars)}" in s.claim
    assert bool(s.top_pairs) == (num_vars > 1)
    bases = ctx.load_bases(srs[:circ.n + 3])
    wpk, pk = equal_keys(ctx, bases, circ, num_vars)
    if circ.witness is not None:  # up to 2^24 + 1 variables (512 MiB): proved from a host vector, staged
        assert circ.witness.shape == (num_vars, 4)
        same_proofs(ctx, wpk, pk, circ, 0x1D + num_vars)
    free(wpk, pk, bases)


# ---- keys and proofs at every domain size, and the cycle shapes at the service's sizes -------------------------------
@pytest.mark.parametrize("log_n", range(2, LOG_MAX + 1))
def test_synthetic_keys_and_proofs(ctx, oracle, srs, tau, log_n):
    n = 1 << log_n
    circ = ws.dense(log_n, num_inputs=min(17, n // 2), seed=0x5100 + log_n).circ
    bases = ctx.load_bases(srs[:n + 3])
    wpk, pk = equal_keys(ctx, bases, circ)
    proof, bl = same_proofs(ctx, wpk, pk, circ, 0xA0 + log_n)
    if log_n == 16:  # the oracle's key and proof
        opk = oracle.plonk_preprocess(log_n, circ.selectors, wiring_permutation(circ.wire_vars), circ.k, srs[:n + 3])
        assert (pk.selector_comms == opk["selector_comms"]).all() and (pk.sigma_comms == opk["sigma_comms"]).all()
        rc, oproof, _, _ = oracle.plonk_prove(log_n, circ.num_inputs, circ.k, opk, expand(circ), circ.pub_inputs, bl,
                                              srs[:n + 3])
        assert rc == 0 and bytes(oproof) == bytes(proof)
    elif log_n == 17:  # the oracle's verifier
        opk = {"selector_comms": pk.selector_comms, "sigma_comms": pk.sigma_comms}
        op = oracle.PlonkProof.from_buffer_copy(bytes(proof))
        assert oracle.plonk_verify_known_tau(log_n, circ.num_inputs, circ.k, opk, circ.pub_inputs, op, tau)
    free(wpk, pk, bases)


@pytest.mark.parametrize("log_n", [16, 17])
@pytest.mark.parametrize("shape", ["one_variable", "each_once_descending", "block_boundary_pairs", "stride_n"])
def test_cycle_shapes_at_full_size(ctx, srs, shape, log_n):
    s = getattr(ws, shape)(log_n)
    circ = s.circ
    assert circ.n * 5 == circ.wire_vars.size and circ.num_inputs == 0
    if shape == "block_boundary_pairs":  # a two-position variable across every block boundary of k_wiring_cycles
        sv = np.sort(circ.wire_vars.reshape(-1))
        assert all(sv[t - 1] == sv[t] for t in range(ws.CYCLE_THREADS, sv.size, ws.CYCLE_THREADS))
    bases = ctx.load_bases(srs[:circ.n + 3])
    wpk, pk = equal_keys(ctx, bases, circ)
    same_proofs(ctx, wpk, pk, circ, 0x16 + log_n)
    free(wpk, pk, bases)


# ---- witness pointer kinds -------------------------------------------------------------------------------------------
KINDS = ["numpy", "pinned", "device", "device+16", "device+8", "managed"]


class Sources:
    """Witness vectors as every pointer kind the prover takes: a numpy array, a pinned tensor, an aligned device tensor,
    a device pointer 16 bytes in (read in place), a device pointer 8 bytes in (staged, public inputs read back) and
    managed memory, allocated through the libcudart torch has loaded (the same device and unified address space as
    the prover's).  The offset pointers sit in allocations one element longer than the vector, so the vector ends
    inside them.  Every buffer lives until close()."""

    def __init__(self):
        import torch
        torch.cuda.init()
        self._rt = C.CDLL("libcudart.so.12")
        self._keep, self._managed = [], []

    def pointer(self, witness, kind):
        import torch
        arr = np.ascontiguousarray(witness)
        self._keep.append(arr)
        if kind == "numpy":
            return arr
        if kind == "managed":
            p = C.c_void_p()
            assert self._rt.cudaMallocManaged(C.byref(p), C.c_size_t(arr.nbytes), C.c_uint(1)) == 0  # AttachGlobal
            self._managed.append(p.value)
            assert self._rt.cudaDeviceSynchronize() == 0
            C.memmove(p.value, arr.ctypes.data, arr.nbytes)
            return p.value
        w = torch.from_numpy(arr.view(np.int64).reshape(-1))
        if kind == "pinned":
            t, off = w.pin_memory(), 0
        else:
            off = {"device": 0, "device+16": 2, "device+8": 1}[kind]  # in int64 elements
            t = torch.zeros(w.numel() + (4 if off else 0), dtype=torch.int64, device="cuda")
            t[off:off + w.numel()] = w.cuda()
            torch.cuda.synchronize()
        self._keep.append(t)
        p = t.data_ptr() + 8 * off
        assert p % 16 == (8 if kind == "device+8" else 0), kind  # in place from 16-byte alignment on
        return p

    def close(self):
        for p in self._managed:
            self._rt.cudaFree(C.c_void_p(p))
        self._managed = []


def test_pointer_kinds_in_one_batch(ctx, srs):
    circ = ws.public_inputs(8, 5, shared=True, zero=True).circ
    bases = ctx.load_bases(srs[:circ.n + 3])
    wpk, pk = equal_keys(ctx, bases, circ)
    src = Sources()
    try:
        ptrs = [src.pointer(circ.witness, kind) for kind in KINDS]
        bls = [synth.splitmix_blinders(0x9000 + i) for i in range(len(KINDS))]
        want = [from_table(ctx, pk, circ, b) for b in bls]
        proofs, hints, st, pubs, chs = PlonkKzgSnark.prove_witness_batch(ctx, wpk, ptrs, bls, link_hints=True,
                                                                         want_challenges=True)
        assert st == [0] * len(KINDS)
        for i, kind in enumerate(KINDS):
            assert (bytes(proofs[i]), hints[i].linking_wire_poly.tobytes(), chs[i].tobytes()) == want[i], kind
            assert (pubs[i] == circ.pub_inputs).all(), kind
            got, pub = from_witness(ctx, wpk, ptrs[i], bls[i])  # the single proof from the same pointer
            assert got == want[i] and (pub == circ.pub_inputs).all(), kind
    finally:
        src.close()
    free(wpk, pk, bases)


# ---- past one gather group -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("k", [65, 130])
def test_batch_past_one_gather_group(ctx, srs, monkeypatch, k):
    """One prover call of 65 / 130 proofs gathers them in groups of 64 (the p0 loop of prove()): statuses and bytes
    equal the single proofs.  Every item has its own witness vector (so an item reading another's is seen), the pointer
    kinds are mixed, and the items at 63, 64 and 129 do not satisfy the circuit."""
    circ = ws.dense(5, num_inputs=2, seed=0x65).circ
    bases = ctx.load_bases(srs[:circ.n + 3])
    wpk, pk = equal_keys(ctx, bases, circ)
    bad_at = {63, 64, 129} & set(range(k))
    circs = [ws.with_witness(circ, w) for w in ws.dense_witnesses(circ, k, seed=k)]
    wits = [unsatisfying(c) if i in bad_at else c.witness for i, c in enumerate(circs)]
    src = Sources()
    try:
        ptrs = [src.pointer(w, KINDS[i % len(KINDS)]) for i, w in enumerate(wits)]
        bls = [synth.splitmix_blinders(0x6500 + i) for i in range(k)]
        want = [None if i in bad_at else from_table(ctx, pk, circs[i], bls[i]) for i in range(k)]
        for chunk in (str(k), None):  # one call of k proofs, then the default chunking (at most 64 per call)
            if chunk:
                monkeypatch.setenv("B200_PROVE_BATCH_CHUNK", chunk)
            else:
                monkeypatch.delenv("B200_PROVE_BATCH_CHUNK")
            proofs, hints, st, pubs, chs = PlonkKzgSnark.prove_witness_batch(ctx, wpk, ptrs, bls, link_hints=True,
                                                                             want_challenges=True)
            assert st == [UNSAT if i in bad_at else 0 for i in range(k)], chunk
            for i in range(k):
                if i in bad_at:
                    assert bytes(proofs[i]) == bytes(len(want[0][0])) and hints[i] is None, (chunk, i)
                else:
                    assert (bytes(proofs[i]), hints[i].linking_wire_poly.tobytes(), chs[i].tobytes()) == want[i], (chunk, i)
                    assert (pubs[i] == circs[i].pub_inputs).all(), (chunk, i)
    finally:
        src.close()
    free(wpk, pk, bases)


# ---- staging growth under graphs --------------------------------------------------------------------------------------
def test_staging_growth_under_replayed_graphs(srs):
    """Key A is proved eager, captured and replayed; key B (same n, 128n variables) stages a witness longer than the
    NTT scratch its context holds (witness_shapes.staging_floor: 78n at this size, from preprocess), which grows it —
    A's graphs hold the old address and must be captured again; then B replays.  A fresh context holding only keys of
    this size, so that the growth is B's."""
    import renegade_b200 as rb
    c = rb.Context(0)
    try:
        c.use_graphs(True)
        a = ws.dense(10, num_inputs=3, seed=0xA).circ
        sb = ws.unused_variables(10)
        b = sb.circ
        assert a.n == b.n and a.num_vars <= ws.staging_floor(a.log_n) < sb.num_vars  # A's witness fits, B's does not
        bases = c.load_bases(srs[:a.n + 3])
        wa, pa = equal_keys(c, bases, a)
        wb, pb = equal_keys(c, bases, b)
        bls = [synth.splitmix_blinders(0x4700 + i) for i in range(9)]
        want_a = {i: from_table(c, pa, a, bls[i]) for i in (0, 1, 2, 4, 6)}
        want_b = {i: from_table(c, pb, b, bls[i]) for i in (3, 5, 7)}
        g0 = c.graph_launches()
        for i in (0, 1, 2):                       # A: eager, captured, replayed
            assert from_witness(c, wa, a.witness, bls[i])[0] == want_a[i], i
        assert c.graph_launches() - g0 == 2 * 7
        for i, (key, circ, want) in zip((3, 4, 5, 6, 7), [(wb, b, want_b), (wa, a, want_a)] * 2 + [(wb, b, want_b)]):
            got, pub = from_witness(c, key, circ.witness, bls[i])
            assert got == want[i], i
            assert (pub == circ.pub_inputs).all(), i
        free(wa, pa, wb, pb, bases)
    finally:
        c.close()


# ---- public-input extremes --------------------------------------------------------------------------------------------
PUBLIC = [("every_row_public", 5), ("every_row_public", 10), ("shared_and_zero", 6), ("shared_and_zero", 13),
          ("inputs_4097", 13)]


@pytest.mark.parametrize("case,log_n", PUBLIC)
def test_public_input_extremes(ctx, oracle, srs, srs_2_16_g2, case, log_n):
    if case == "every_row_public":
        s = ws.every_row_public(log_n)
        assert s.circ.num_inputs == s.circ.n
    elif case == "shared_and_zero":
        s = ws.public_inputs(log_n, 9, shared=True, zero=True)
    else:
        s = ws.public_inputs(log_n, 4097)
        assert s.circ.num_inputs > 4096  # one proof's public-input denominators span two k_block_inverse blocks
    circ = s.circ
    bases = ctx.load_bases(srs[:circ.n + 3])
    wpk, pk = equal_keys(ctx, bases, circ)
    proof, bl = same_proofs(ctx, wpk, pk, circ, 0x70 + log_n)
    pub = circ.pub_inputs
    if case == "inputs_4097":  # = the oracle's proof
        opk = oracle.plonk_preprocess(log_n, circ.selectors, wiring_permutation(circ.wire_vars), circ.k, srs[:circ.n + 3])
        rc, oproof, _, _ = oracle.plonk_prove(log_n, circ.num_inputs, circ.k, opk, expand(circ), circ.pub_inputs, bl,
                                              srs[:circ.n + 3])
        assert rc == 0 and bytes(oproof) == bytes(proof)
    vk = VerifyingKey.from_proving_key(wpk, *srs_2_16_g2)
    wrong = pub.copy()
    wrong[-1, 0] ^= 1
    assert PlonkKzgSnark.verify(vk, pub, proof) and not PlonkKzgSnark.verify(vk, wrong, proof)
    for items in ([pub], [wrong], [pub, wrong], [wrong, pub]):
        expect = [p is pub for p in items]
        ok, verdicts = PlonkKzgSnark.batch_verify(ctx, [vk] * len(items), items, [proof] * len(items))
        assert verdicts == expect and ok == all(expect), (case, len(items))
        assert PlonkKzgSnark.verify_each(ctx, [vk] * len(items), items, [proof] * len(items)) == expect, (case, len(items))
    free(wpk, pk, bases)


# ---- refusals ---------------------------------------------------------------------------------------------------------
def test_num_vars_limits(ctx, srs):
    s = ws.index_width((1 << 32) - 1)
    circ = s.circ
    bases = ctx.load_bases(srs[:circ.n + 3])
    with pytest.raises(_lib.B200Error) as err:
        PlonkKzgSnark.preprocess_wiring(ctx, bases, circ.log_n, 0, circ.selectors, circ.wire_vars, 1 << 32, circ.k)
    assert err.value.code == INVALID
    wpk, pk = equal_keys(ctx, bases, circ, (1 << 32) - 1)  # the widest index: a key, never a proof (no such witness exists)
    assert wpk.num_vars == (1 << 32) - 1
    free(wpk, pk)
    d = ws.dense(4, num_inputs=2, seed=0x32).circ
    wpk, pk = equal_keys(ctx, bases, d)
    same_proofs(ctx, wpk, pk, d, 0x32)  # the context keeps proving
    free(wpk, pk, bases)
