"""GPU: the prover above 2^17, where its chunked scans (CH = 16) take their deepest shapes — the grand product's 5-level
scan in full at 2^20 and its 6-level scan from 2^21, the opening Horner scans at 6 levels — and its commitments of
n + 2 and n + 3 coefficients run through the largest SRS window plans.  Circuits from tests/large_domains.py.

- 2^18 and 2^20: keys and proofs byte for byte = the oracle (every commitment, evaluation, challenge and the linking
  polynomial), from the table and from the witness vector, eagerly and from replayed graphs; at 2^20 also batches of 3
  (one MSM of 15 wire commitments) in the chunk the library's rule chooses and in chunks of 1, a batch of 6 split by
  the memory budget, and a link proof, which verifies and is rejected under a shifted layout or with swapped points.
- 2^21 and 2^22 (the largest domain whose key and proof fit an 80 GB H100): the oracle is too slow to prove there, so
  every entry point is held to the same bytes and the proof to the oracle's known-τ verifier and the product's three
  verifiers; a tampered evaluation and a changed public input are rejected by all four.  At 2^21 an unsatisfied witness
  (a gate, and a copy across z's wrap) is refused eagerly and from replayed graphs.

Each size runs on a context of its own and skips, with the numbers, when the GPU has less free memory than
`large_domains.footprint_bytes` × 1.15 for the keys its tests hold at once; each batch skips likewise on the batch
buffers its largest possible chunk adds.  The memory each size used (free memory before minus after: meaningful on an
otherwise idle GPU) is printed next to the estimate."""
import gc
import time

import numpy as np
import pytest
import torch

import large_domains as ld
import renegade_b200 as rb
from renegade_b200 import _lib, synth
from renegade_b200.backend import B200Proof, GroupLayout, PlonkKzgSnark, VerifyingKey, link_proofs, verify_link_proof

pytestmark = pytest.mark.gpu

TAU = 0x0B5E55ED1A2B3C4D5E6F708192A3B4C5D6E7F8091A2B3C4D5E6F708192A3B4C5
SLACK = 1.15
NAMES = ["wire_comm"] * 40 + ["z_comm"] * 8 + ["quot_comm"] * 40 + ["opening"] * 8 + ["shifted"] * 8 + \
        ["wire_eval"] * 20 + ["sigma_eval"] * 16 + ["z_next"] * 4
_LIVE = []


def _free():
    gc.collect()
    torch.cuda.empty_cache()
    return torch.cuda.mem_get_info()


class Size:
    """One domain size on a context of its own: circuit, known-τ SRS, (H, τH), and the device memory it has used."""

    def __init__(self, oracle, pyoracle, g2_raw, log_n, seed, keys):
        import bn254_pairing_py as pr
        for other in list(_LIVE):
            other.close()
        self.log_n, self.n = log_n, 1 << log_n
        free, total = _free()
        need = int(ld.footprint_bytes(log_n, keys=keys) * SLACK)  # the most the tests of this size hold at once
        if free < need:
            pytest.skip(f"2^{log_n}: {need >> 20} MiB wanted ({keys} keys, estimate x {SLACK}), {free >> 20} of "
                        f"{total >> 20} MiB free")
        t0 = time.time()
        self.circ = ld.big_circuit(log_n, seed=seed)
        self.tau = oracle.int_to_limbs(pyoracle.to_mont(TAU % pyoracle.R, pyoracle.R))
        self.srs = oracle.srs_from_tau(self.tau, self.n + 3)
        h = g2_raw[0]
        tau_h = pr.encode_g2_mont(pr.g2_mul(pr.decode_g2_mont(h.tobytes(), 0), TAU % pr.R))
        self.g2 = (h, np.frombuffer(tau_h, dtype=np.uint64).copy())
        print(f"\n2^{log_n}: circuit and SRS on the host in {time.time() - t0:.1f} s; {free >> 20} of {total >> 20} MiB free, "
              f"{need >> 20} MiB wanted", flush=True)
        self.ctx = self.bases = None
        self.keys = []
        self.peak = 0
        self.results = {}
        self.batch_chunk = 0  # the largest chunk the context's batch buffers have held
        self.keys_held = keys
        _LIVE.append(self)
        self.open()

    def open(self):
        """A fresh context with the SRS loaded."""
        self.close_ctx()
        self.batch_chunk = 0
        self.free0 = _free()[0]
        self.ctx = rb.Context(0)
        self.bases = self.ctx.load_bases(self.srs)

    def measure(self, what):
        """Free memory before the context minus free memory now: the context's use on an otherwise idle GPU (other
        processes' allocations in between count too)."""
        used = self.free0 - torch.cuda.mem_get_info()[0]
        self.peak = max(self.peak, used)
        print(f"2^{self.log_n} {what}: {used / 2**30:.2f} GiB in use on the device", flush=True)
        return used

    def key(self, wiring=False):
        c = self.circ
        if wiring:
            pk = PlonkKzgSnark.preprocess_wiring(self.ctx, self.bases, self.log_n, c.num_inputs, c.selectors, c.wire_vars,
                                                 c.num_vars, c.k)
        else:
            pk = PlonkKzgSnark.preprocess(self.ctx, self.bases, self.log_n, c.num_inputs, c.selectors, c.perm, c.k)
        self.keys.append(pk)
        return pk

    def vk(self, pk):
        return VerifyingKey.from_proving_key(pk, *self.g2)

    def close_ctx(self):
        for pk in self.keys:
            pk.free()
        self.keys = []
        if self.bases is not None:
            self.bases.free()
            self.bases = None
        if self.ctx is not None:
            self.ctx.close()
            self.ctx = None
            torch.cuda.synchronize()

    def close(self):
        est = ld.footprint_parts(self.log_n, keys=self.keys_held)
        print(f"2^{self.log_n}: peak {self.peak / 2**30:.2f} GiB measured, estimate {sum(est.values()) / 2**30:.2f} GiB "
              f"({', '.join(f'{k} {v / 2**30:.2f}' for k, v in est.items())})", flush=True)
        self.close_ctx()
        if self in _LIVE:
            _LIVE.remove(self)


def _size(request, oracle, pyoracle, g2_raw, log_n, seed, keys):
    s = Size(oracle, pyoracle, g2_raw, log_n, seed, keys)
    request.addfinalizer(s.close)
    return s


@pytest.fixture(scope="module")
def size18(request, oracle, pyoracle, g2_raw):
    return _size(request, oracle, pyoracle, g2_raw, 18, 0x18, keys=2)


@pytest.fixture(scope="module")
def size20(request, oracle, pyoracle, g2_raw):
    return _size(request, oracle, pyoracle, g2_raw, 20, 0x20, keys=2)


@pytest.fixture(scope="module")
def size21(request, oracle, pyoracle, g2_raw):
    return _size(request, oracle, pyoracle, g2_raw, 21, 0x21, keys=1)


@pytest.fixture(scope="module")
def size22(request, oracle, pyoracle, g2_raw):
    return _size(request, oracle, pyoracle, g2_raw, 22, 0x22, keys=1)


def assert_same_proof(ours, theirs, what):
    a, b = ours.to_array(), theirs.to_array()
    diff = sorted({NAMES[i] for i in range(len(NAMES)) if a[i] != b[i]})
    assert not diff, (what, diff)


def batch_bytes(s, chunk):
    """The batch buffers of a context whose batches ran in chunks of up to `chunk` proofs (0: none yet)."""
    if chunk == 0:
        return 0
    return sum(v for k, v in ld.footprint_parts(s.log_n, chunk, batch=True).items() if k.startswith("batch_"))


def chunk_rule(s, pk, k, free_b):
    """prove_batch_chunk (plonk.cu) restated: half of the free memory plus the batch buffers the context already has
    (they are reused) over one proof's workspace, NTT scratches and MSM scratch of its NW commitments; at most 64; and
    the MSM's 32-bit entry index, n * digits * NW * chunk < 2^32.  Returns (chunk, per_proof, idx_cap)."""
    c = ld.constants()
    n = s.n
    m = ld.cosets(s.log_n, c) * n
    plan = s.bases.plan
    msm_per_commit = n * plan["digits"] * 4 * 2 + (plan["physical_windows"] << (plan["window_bits"] - 1)) * 128 * 4
    per_proof = (ld.workspace_elems(n, 1, c) + 6 * m + max(c["STAGE_PER_M"] * m, pk.num_vars)) * 32 + c["NW"] * msm_per_commit
    caps = 0
    if s.batch_chunk:
        q = s.batch_chunk
        caps = (ld.workspace_elems(n, q, c) + q * max(c["STAGE_PER_M"] * m, pk.num_vars) + q * 6 * m) * 32
    budget = (free_b + caps) // 2
    idx_cap = (1 << 32) // (n * plan["digits"] * c["NW"]) - 1
    return max(1, min(k, 64, budget // per_proof, idx_cap)), per_proof, idx_cap


def run_batch(s, pk, wires, pub, bls, forced=None, **kw):
    """prove_batch of len(bls) items, gated on the memory of the largest chunk it can take.  The chunk the library chose
    is read from the MSM launch count (4 batched MSMs per prover call) and must be the rule's for free memory within
    5 % of the reading taken just before the call (the library takes its own, a moment later).  Returns (result, chunk)."""
    k = len(bls)
    free_b, total = _free()
    if forced:
        chunks = {min(forced, k)}
    else:
        chunks = {chunk_rule(s, pk, k, int(free_b * f))[0] for f in (0.95, 1.0, 1.05)}
    need = int(SLACK * max(0, batch_bytes(s, max(chunks)) - batch_bytes(s, s.batch_chunk)))
    if free_b < need:
        pytest.skip(f"2^{s.log_n} batch of {k} in chunks of {max(chunks)}: {need >> 20} MiB more wanted, {free_b >> 20} of "
                    f"{total >> 20} MiB free")
    _, per_proof, idx_cap = chunk_rule(s, pk, k, free_b)
    s.ctx.msm_timing(True)
    s.ctx.msm_timing_totals(reset=True)
    res = PlonkKzgSnark.prove_batch(s.ctx, pk, [wires] * k, [pub] * k, bls, **kw)
    launches = s.ctx.msm_timing_totals()["launches"]
    s.ctx.msm_timing(False)
    chosen = [q for q in sorted(chunks) if launches == 4 * -(-k // q)]
    print(f"2^{s.log_n} batch of {k}: {launches:.0f} MSM launches, rule's chunks {sorted(chunks)} (per proof {per_proof >> 20} "
          f"MiB, {free_b >> 20} MiB free, idx_cap {idx_cap})", flush=True)
    assert chosen, (launches, sorted(chunks))
    s.batch_chunk = max(s.batch_chunk, chosen[-1])
    assert list(res[2]) == [0] * k
    s.measure(f"batch of {k} in chunks of {chosen[-1]}")
    return res, chosen[-1]


# ---- 2^18 and 2^20: the oracle's bytes ----------------------------------------------------------------------------------
def oracle_parity(s, oracle):
    c, ctx, log_n = s.circ, s.ctx, s.log_n
    pk = s.key()
    t0 = time.time()
    opk = oracle.plonk_preprocess(log_n, c.selectors, c.perm, c.k, s.srs)
    t_pre = time.time() - t0
    assert (pk.selector_comms == opk["selector_comms"]).all() and (pk.sigma_comms == opk["sigma_comms"]).all()
    bl = synth.splitmix_blinders(0xB16 + log_n)
    proof, hint, ch = PlonkKzgSnark.prove_with_link_hint(ctx, pk, c.wires, c.pub_inputs, bl, want_challenges=True)
    t0 = time.time()
    rc, oproof, och, olink = oracle.plonk_prove(log_n, c.num_inputs, c.k, opk, c.wires, c.pub_inputs, bl, s.srs, True)
    t_prove = time.time() - t0
    print(f"2^{log_n}: oracle preprocess {t_pre:.1f} s, prove {t_prove:.1f} s (CPU threads: {oracle.num_threads()})", flush=True)
    assert rc == 0
    assert_same_proof(proof, oproof, "prove")
    assert (ch.reshape(-1) == np.frombuffer(bytes(och), dtype=np.uint64)).all()
    assert (hint.linking_wire_poly == olink).all()
    s.measure("key and one proof")
    # a second proof of the key with other blinders, captured and then replayed as graphs: = oracle
    bl2 = synth.splitmix_blinders(0xB17 + log_n)
    g0 = ctx.graph_launches()
    replayed = [PlonkKzgSnark.prove_with_link_hint(ctx, pk, c.wires, c.pub_inputs, bl2) for _ in range(2)]
    assert ctx.graph_launches() > g0
    rc, oproof2, _, olink2 = oracle.plonk_prove(log_n, c.num_inputs, c.k, opk, c.wires, c.pub_inputs, bl2, s.srs, True)
    assert rc == 0
    for p2, h2 in replayed:
        assert_same_proof(p2, oproof2, "replayed graphs")
        assert (h2.linking_wire_poly == olink2).all()
    opk_v = {"selector_comms": pk.selector_comms, "sigma_comms": pk.sigma_comms}
    assert oracle.plonk_verify_known_tau(log_n, c.num_inputs, c.k, opk_v, c.pub_inputs, oproof, s.tau)
    # the same circuit as wiring + witness vector: same key, same bytes
    wpk = s.key(wiring=True)
    assert (wpk.selector_comms == pk.selector_comms).all() and (wpk.sigma_comms == pk.sigma_comms).all()
    wproof, whint, wpub, wch = PlonkKzgSnark.prove_witness(ctx, wpk, c.witness, bl, want_challenges=True)
    assert_same_proof(wproof, oproof, "prove_witness")
    assert (wpub == c.pub_inputs).all() and (wch == ch).all() and (whint.linking_wire_poly == olink).all()
    s.measure("two keys and five proofs")
    wpk.free()
    s.keys.remove(wpk)
    s.results.update(pk=pk, opk=opk, bl=bl, bl2=bl2, proof=proof, hint=hint, proof2=replayed[0][0], hint2=replayed[0][1])


def test_2_18_oracle_bytes(size18, oracle):
    oracle_parity(size18, oracle)


def test_2_20_oracle_bytes(size20, oracle):
    oracle_parity(size20, oracle)


def test_2_20_batches(size20, monkeypatch):
    """prove_batch of 3 witnesses (one MSM of 15 wire commitments: the device-Horner epilogue) in the chunk the library's
    rule chooses and in chunks of 1, then of 6, which the memory budget splits (at most 4 proofs of 2^20 fit half of an
    80 GB card beside the key): every item = the single proof of the same witness and blinders.  The 32-bit entry cap
    (62 proofs at 2^20) is not reached: no 80 GB card holds that many 2^20 proofs at once."""
    s = size20
    if "pk" not in s.results:
        pytest.skip("needs test_2_20_oracle_bytes")
    c, ctx, pk, r = s.circ, s.ctx, s.results["pk"], s.results
    bl3 = synth.splitmix_blinders(0xB18 + s.log_n)
    p3, h3 = PlonkKzgSnark.prove_with_link_hint(ctx, pk, c.wires, c.pub_inputs, bl3)
    singles = [(r["proof"], r["hint"]), (r["proof2"], r["hint2"]), (p3, h3)]
    bls = [r["bl"], r["bl2"], bl3]
    for forced, k in ((None, 3), (1, 3), (None, 6)):
        if forced:
            monkeypatch.setenv("B200_PROVE_BATCH_CHUNK", str(forced))
        else:
            monkeypatch.delenv("B200_PROVE_BATCH_CHUNK", raising=False)
        (proofs, hints, _), chunk = run_batch(s, pk, c.wires, c.pub_inputs, (bls * 2)[:k], forced, link_hints=True)
        if k == 6:
            assert chunk < k, "the budget did not split a batch of 6 proofs of 2^20"
        for i, (bp, bh) in enumerate(zip(proofs, hints)):
            sp, sh = singles[i % 3]
            assert_same_proof(bp, sp, f"batch of {k}, item {i}, chunk {chunk}")
            assert (bh.linking_wire_poly == sh.linking_wire_poly).all()


def test_2_20_link(size20, oracle):
    """A link proof between two 2^20 proofs of the same circuit and witness with other blinders (so the linking
    polynomials agree on H and differ off it) over GroupLayout(20, n - 8, 8): the last 8 rows, the last at n - 1 — the
    layout synth's link= places at alignment 20, here over wire 0 of the circuit's own rows rather than link gates.
    = oracle, accepted by the product's and the oracle's link verifiers; under a layout one row lower, or with its two
    points swapped, the proof is rejected by both."""
    s = size20
    if "pk" not in s.results:
        pytest.skip("needs test_2_20_oracle_bytes")
    h1, h2 = s.results["hint"], s.results["hint2"]
    layout = GroupLayout(alignment=20, offset=s.n - 8, size=8)
    assert not (h1.linking_wire_poly == h2.linking_wire_poly).all()
    lp, eta = link_proofs(s.ctx, s.bases, h1, h2, layout)
    rc, olp, oeta = oracle.plonk_link(h1.linking_wire_poly, h2.linking_wire_poly, h1.linking_wire_comm, h2.linking_wire_comm,
                                      layout.alignment, layout.offset, layout.size, s.srs)
    assert rc == 0 and (lp.to_array() == olp.to_array()).all() and (eta == oeta).all()
    assert verify_link_proof(h1.linking_wire_comm, h2.linking_wire_comm, lp, layout, *s.g2)
    assert oracle.plonk_link_verify_known_tau(h1.linking_wire_comm, h2.linking_wire_comm, layout.alignment, layout.offset,
                                              layout.size, oracle.LinkProof.from_buffer_copy(bytes(lp)), s.tau)
    shifted = GroupLayout(layout.alignment, layout.offset - 1, layout.size)
    swapped = type(lp).from_buffer_copy(bytes(lp))
    swapped.quotient_commitment[:], swapped.opening_proof[:] = list(lp.opening_proof), list(lp.quotient_commitment)
    for proof, lay in ((lp, shifted), (swapped, layout)):
        assert not verify_link_proof(h1.linking_wire_comm, h2.linking_wire_comm, proof, lay, *s.g2)
        assert not oracle.plonk_link_verify_known_tau(h1.linking_wire_comm, h2.linking_wire_comm, lay.alignment, lay.offset,
                                                      lay.size, oracle.LinkProof.from_buffer_copy(bytes(proof)), s.tau)


# ---- 2^21 and 2^22: the device against itself and the verifiers --------------------------------------------------------
def verdicts(s, oracle, pk, pub, proof):
    """(oracle known-τ, b200_plonk_verify, b200_plonk_batch_verify, b200_plonk_verify_each)"""
    c = s.circ
    opk = {"selector_comms": pk.selector_comms, "sigma_comms": pk.sigma_comms}
    vk = s.vk(pk)
    ok_b, v_b = PlonkKzgSnark.batch_verify(s.ctx, [vk], [pub], [proof])
    return (oracle.plonk_verify_known_tau(s.log_n, c.num_inputs, c.k, opk, pub, oracle.PlonkProof.from_buffer_copy(bytes(proof)),
                                          s.tau),
            PlonkKzgSnark.verify(vk, pub, proof), ok_b and v_b == [True], PlonkKzgSnark.verify_each(s.ctx, [vk], [pub], [proof]) == [True])


def self_consistency(s, oracle):
    c, ctx = s.circ, s.ctx
    bl = synth.splitmix_blinders(0xB19 + s.log_n)
    pk = s.key()
    proofs = [PlonkKzgSnark.prove_with_link_hint(ctx, pk, c.wires, c.pub_inputs, bl)[0]]  # eager
    g0 = ctx.graph_launches()
    proofs += [PlonkKzgSnark.prove_with_link_hint(ctx, pk, c.wires, c.pub_inputs, bl)[0] for _ in range(2)]  # captured, replayed
    assert ctx.graph_launches() > g0
    ref = proofs[0]
    for i, p in enumerate(proofs):
        assert_same_proof(p, ref, f"proof {i}")
    assert verdicts(s, oracle, pk, c.pub_inputs, ref) == (True,) * 4
    bad = B200Proof.from_buffer_copy(bytes(ref))
    bad.wires_evals[2][0] ^= 1
    assert verdicts(s, oracle, pk, c.pub_inputs, bad) == (False,) * 4
    wrong = c.pub_inputs.copy()
    wrong[-1] = c.pub_inputs[0] if (c.pub_inputs[0] != c.pub_inputs[-1]).any() else c.pub_inputs[1]
    assert verdicts(s, oracle, pk, wrong, ref) == (False,) * 4
    s.measure("key and three proofs")
    pk.free()
    s.keys.remove(pk)
    wpk = s.key(wiring=True)
    wproof, _, wpub = PlonkKzgSnark.prove_witness(ctx, wpk, c.witness, bl)
    assert_same_proof(wproof, ref, "prove_witness")
    assert (wpub == c.pub_inputs).all()
    s.measure("wiring key and its proof")
    # a batch of 2 on a fresh context: the batch buffers come on top of the single prover's otherwise
    s.open()
    pk = s.key()
    bl2 = synth.splitmix_blinders(0xB1A + s.log_n)
    (proofs, _, _), chunk = run_batch(s, pk, c.wires, c.pub_inputs, [bl, bl2])
    assert_same_proof(proofs[0], ref, f"batch item 0, chunk {chunk}")
    assert verdicts(s, oracle, pk, c.pub_inputs, proofs[1]) == (True,) * 4
    assert bytes(proofs[1]) != bytes(ref)


def test_2_21_self_consistent(size21, oracle):
    self_consistency(size21, oracle)


def test_2_21_unsatisfied(size21, oracle):
    """A gate violation on one row (its error polynomial is the indicator of that row: degree n - 1, for round 3's
    degree check) and a copy-only violation on the ends cycle at row n - 1, where z wraps: B200_ERR_UNSATISFIED from
    the key's first, eager call and from replayed graphs; after each refusal the honest proof = its earlier bytes."""
    s = size21
    s.open()
    c, ctx = s.circ, s.ctx
    n, wv = s.n, c.wire_vars
    counts = np.bincount(wv.reshape(-1))
    row = next(r for r in sorted(c.gate_rows) if r > n // 2 and c.gate_rows[r] == "hash")
    col = next(i for i in (1, 2, 3) if counts[wv[i, row]] == 1)   # a gate input no copy constraint reaches
    gate_bad = c.wires.copy()
    gate_bad[col, row] = ld.random_fr(np.random.default_rng(1), 1)[0]
    copy_bad = c.wires.copy()
    assert wv[1, n - 1] == c.boundary["ends"][0] and not c.selectors[:, n - 1].any()
    copy_bad[1, n - 1] = ld.random_fr(np.random.default_rng(2), 1)[0]
    bl = synth.splitmix_blinders(0xBAD)
    pk = s.key()

    def refused(wires):
        with pytest.raises(_lib.B200Error) as ei:
            PlonkKzgSnark.prove_with_link_hint(ctx, pk, wires, c.pub_inputs, bl)
        assert ei.value.code == _lib.B200_ERR_UNSATISFIED, ei.value

    refused(gate_bad)                                   # the key's first call: eager
    ref = PlonkKzgSnark.prove_with_link_hint(ctx, pk, c.wires, c.pub_inputs, bl)[0]
    assert verdicts(s, oracle, pk, c.pub_inputs, ref) == (True,) * 4
    for bad in (gate_bad, copy_bad, gate_bad):
        g0 = ctx.graph_launches()
        refused(bad)
        assert ctx.graph_launches() > g0                # refused from replayed graphs
        assert bytes(PlonkKzgSnark.prove_with_link_hint(ctx, pk, c.wires, c.pub_inputs, bl)[0]) == bytes(ref)
    s.measure("unsatisfied witnesses")


def test_2_22_self_consistent(size22, oracle):
    self_consistency(size22, oracle)
