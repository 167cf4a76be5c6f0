"""GPU: the proofs bench.py times, made the way it makes them, equal the proofs the rest of the suite pins to the oracle.

bench.py proves its headline (the 2^16 synthetic circuit, 17 public inputs, known-discrete-log SRS made on the device and
loaded with `load_bases_device`) through a pool of 16 workers with MSM timing switched on before warm-up, so that the
timing events are nodes of every captured prover graph, and passes the wires from device, pinned and pageable memory.
Its MSM figure divides by `msm_timing_totals`.  Here:

  * reference bytes: a fresh context with graphs and timing off (the path test_gpu_plonk.py holds to the oracle at every
    size up to 2^16), and one proof per key against `oracle.plonk_prove` directly;
  * the headline regime in-process: 3 warm-up waves of 16, then 48 proofs (device / pinned / pageable wires, 12 blinder
    sets on several workers each, waited for out of order), every one = its reference bytes, the pool's timing totals
    exactly 4 launches and 13n + 32 pairs per proof; the 2^12 private-settlement statement at width 16 and two
    private-match bundles (5 proofs, 4 link proofs) through the same pool = the single calls;
  * MSM timing toggled between proofs (graphs on and off): same bytes, graphs re-captured with the timing nodes, exact
    counts, phases finite with total >= each phase; `prove_batch` and `link_proofs_batch` timed and counted too;
  * B200_STREAM_PRIORITIES unset / 0 / 1 (read by every context at creation): proofs eager and replayed, a pool with
    timing on, a batch, single and batch link proofs, lone latency- and throughput-plan MSMs = reference or oracle;
  * the switches read once per process (B200_QUAD_ADD, B200_TREE_FANIN_LOG, B200_HOST_HORNER, B200_GRAPHS) and bench's
    CUDA_DEVICE_MAX_CONNECTIONS=32, one subprocess each (tests/regime_driver.py): MSMs of every reduction shape and
    proofs = oracle / reference bytes."""
import json
import math
import os
import re
import subprocess
import sys
from types import SimpleNamespace

import numpy as np
import pytest

import link_layouts as ll
import renegade_b200 as rb
from renegade_b200 import synth
from renegade_b200.backend import GroupLayout, LinkingHint, PlonkKzgSnark, ProverPool, link_proofs, link_proofs_batch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DRIVER = os.path.join(ROOT, "tests", "regime_driver.py")
# bench.py's headline: LOG_N, NUM_INPUTS, CIRCUIT_SEED, SEED_SRS
LOG_N, NUM_INPUTS, CIRCUIT_SEED, SEED_SRS = 16, 17, 0xB200, 0x7A0
N = 1 << LOG_N
N_BLINDERS = 12
WORKERS = 16
# device memory the in-process pool of 16 needs at 2^16 besides what is already allocated (workspaces, NTT and MSM
# scratch of 16 workers, the key and the SRS tables), with room to spare
POOL_BYTES = 16 << 30
SWITCHES = ("B200_QUAD_ADD", "B200_TREE_FANIN_LOG", "B200_HOST_HORNER", "B200_GRAPHS", "B200_STREAM_PRIORITIES")


def pairs_per_proof(n: int) -> int:
    """(point, scalar) pairs of one proof's four commitment MSMs: 5 wires (n + 2), z (n + 3), 5 quotient parts (n + 3),
    the two openings (n + 2)"""
    return 5 * (n + 2) + (n + 3) + 5 * (n + 3) + 2 * (n + 2)


def msm_constant(name: str) -> int:
    with open(os.path.join(ROOT, "renegade_b200", "csrc", "msm.cu")) as f:
        m = re.search(rf"constexpr size_t {name} = \(size_t\)1 << (\d+);|constexpr size_t {name} = (\d+);", f.read())
    assert m, f"msm.cu no longer defines {name}"
    return 1 << int(m.group(1)) if m.group(1) else int(m.group(2))


SMALL_TREE_BUCKETS = msm_constant("kSmallTreeBuckets")
QUAD_TREE_MAX_OUTPUTS = msm_constant("kQuadTreeMaxOutputs")


def serial_level(plan: dict, batch: int = 1, forced: int = 0):
    """(fan-in log a_row, a_col, four lanes per addition) of the serial tree level that msm.cu's tree_shape and
    msm_launch_batch choose for `batch` MSMs of this LATENCY plan with the default B200_QUAD_ADD"""
    c = plan["window_bits"]
    n_buckets = batch * plan["physical_windows"] << (c - 1)
    bits = c - 1
    l = (bits + 1) // 2
    r = bits - l
    a = forced or (2 if n_buckets <= SMALL_TREE_BUCKETS else 3)
    if l - a > 8:
        a = l - 8
    a_row, a_col = min(l, a), min(r, a)
    quad = (n_buckets >> a_row) + (n_buckets >> a_col) <= QUAD_TREE_MAX_OUTPUTS
    return a_row, a_col, quad


# ---- inputs and reference bytes ------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def inputs(oracle, pyoracle):
    from host_circuits import private_settlement as ps
    parties, st = ps.create_witness_statement(1)
    py = pyoracle
    same = [1 + 8 * i for i in range(256)]
    return SimpleNamespace(
        srs=oracle.known_dlog_bases(SEED_SRS, N + 3),
        circuits={"synthetic": synth.synth_circuit(LOG_N, num_inputs=NUM_INPUTS, seed=CIRCUIT_SEED),
                  "settlement": ps.IntentAndBalancePrivateSettlementCircuit.build(parties, st).finalize_for_arithmetization()},
        blinders=np.stack([synth.splitmix_blinders(0xBE7C + i) for i in range(N_BLINDERS)]),
        scalars=oracle.splitmix_fr(0x5CA1A8, N, montgomery=False),
        batch_scalars=np.stack([oracle.splitmix_fr(0x100 + b, 1 << 12, montgomery=False) for b in range(12)]),
        one_base={"same": same,
                  "alt": [v if i % 2 == 0 else py.R - v for i, v in enumerate(same)],
                  "wide": [((1 + 8 * i) << 100) + (1 + 8 * (255 - i)) for i in range(256)]})


@pytest.fixture(scope="module")
def bundle_circuits():
    """bench.py's private-match bundle: the settlement proof (2^12), both parties' INTENT AND BALANCE VALIDITY (2^14) and
    OUTPUT BALANCE VALIDITY (2^13) proofs, and the four link proofs between them"""
    from host_circuits import intent_and_balance_validity as val
    from host_circuits import output_balance_validity as obv
    from host_circuits import private_settlement as ps
    parties, _ = ps.create_witness_statement(seed=61)
    validity = [val.create_witness_statement(seed=70 + i, intent=parties[i].intent, balance=parties[i].input_balance)
                for i in (0, 1)]
    out_validity = [obv.create_witness_statement(80 + i, parties[i].output_balance) for i in (0, 1)]
    parties, statement = ps.create_witness_statement(
        seed=61, linked=[(validity[i][0].new_amount_public_share, validity[i][0].post_match_balance_shares,
                          out_validity[i][0].post_match_balance_shares) for i in (0, 1)])
    cs = ps.IntentAndBalancePrivateSettlementCircuit.build(parties, statement)
    layouts = cs.get_circuit_layout()
    circs = [cs.finalize_for_arithmetization()] + \
            [val.IntentAndBalanceValidityCircuit.build(w, s, layouts).finalize_for_arithmetization() for w, s in validity] + \
            [obv.OutputBalanceValidityCircuit.build(w, s, layouts).finalize_for_arithmetization() for w, s in out_validity]
    plan = [(1 + p, GroupLayout(layouts[g].alignment, layouts[g].offset, layouts[g].size)) for p, g in enumerate(ps.PARTY_LINKS)] + \
           [(3 + p, GroupLayout(layouts[g].alignment, layouts[g].offset, layouts[g].size)) for p, g in enumerate(ps.OUTPUT_LINKS)]
    return circs, plan


def preprocess(ctx, bases, circ):
    return PlonkKzgSnark.preprocess(ctx, bases, circ.log_n, circ.num_inputs, circ.selectors, circ.perm, circ.k)


class References:
    """Proofs of a fresh context with graphs and MSM timing off, by (key, blinder set)."""

    def __init__(self, inputs):
        self.inputs = inputs
        self.ctx = rb.Context(0)
        self.ctx.use_graphs(False)
        self.bases = self.ctx.load_bases(inputs.srs)
        self.pks = {key: preprocess(self.ctx, self.bases, c) for key, c in inputs.circuits.items()}
        self.cache = {}

    def proof(self, key, b):
        """(proof bytes, link polynomial) of circuit `key` with blinder set b"""
        if (key, b) not in self.cache:
            c = self.inputs.circuits[key]
            proof, hint = PlonkKzgSnark.prove_with_link_hint(self.ctx, self.pks[key], c.wires, c.pub_inputs, self.inputs.blinders[b])
            self.cache[key, b] = (bytes(proof), hint.linking_wire_poly)
        return self.cache[key, b]

    def close(self):
        for pk in self.pks.values():
            pk.free()
        self.bases.free()
        self.ctx.close()


@pytest.fixture(scope="module")
def refs(inputs):
    r = References(inputs)
    yield r
    r.close()


@pytest.mark.parametrize("key", ["synthetic", "settlement"])
def test_reference_bytes_equal_the_oracle(inputs, refs, oracle, key):
    c = inputs.circuits[key]
    srs = inputs.srs[:c.n + 3]
    opk = oracle.plonk_preprocess(c.log_n, c.selectors, c.perm, c.k, srs)
    assert (refs.pks[key].selector_comms == opk["selector_comms"]).all() and (refs.pks[key].sigma_comms == opk["sigma_comms"]).all()
    rc, oproof, _, olink = oracle.plonk_prove(c.log_n, c.num_inputs, c.k, opk, c.wires, c.pub_inputs, inputs.blinders[0], srs, True)
    assert rc == 0
    proof, link = refs.proof(key, 0)
    assert proof == bytes(oproof) and (link == olink).all()


# ---- the headline regime, in-process --------------------------------------------------------------------------------
def test_headline_regime_pool_of_16(inputs, refs, bundle_circuits):
    import torch
    free, total = torch.cuda.mem_get_info()
    if free < POOL_BYTES:
        pytest.skip(f"a pool of {WORKERS} at 2^{LOG_N} wants {POOL_BYTES >> 20} MiB free, the GPU has {free >> 20} of "
                    f"{total >> 20} MiB free")
    circ = inputs.circuits["synthetic"]
    pool = ProverPool(0, workers=WORKERS)
    try:
        ctxs = [pool.context(i) for i in range(WORKERS)]
        ctx = ctxs[0]
        d_srs = torch.empty((N + 3, 8), dtype=torch.int64, device="cuda")
        torch.cuda.synchronize()
        ctx.known_dlog_bases_device(SEED_SRS, N + 3, d_srs.data_ptr())
        assert (d_srs.cpu().numpy().view(np.uint64) == inputs.srs).all()
        srs = ctx.load_bases_device(d_srs.data_ptr(), N + 3)
        pk = preprocess(ctx, srs, circ)
        assert (pk.selector_comms == refs.pks["synthetic"].selector_comms).all()
        assert (pk.sigma_comms == refs.pks["synthetic"].sigma_comms).all()
        for c in ctxs:  # before warm-up, as bench.py does: the timing events become nodes of every captured graph
            c.msm_timing(True)
        h_w = torch.from_numpy(circ.wires.view(np.int64)).pin_memory()
        d_w = h_w.to("cuda")
        p_w = np.ascontiguousarray(circ.wires, dtype=np.uint64).copy()
        torch.cuda.synchronize()
        wires = {"device": d_w.data_ptr(), "pinned": h_w.data_ptr(), "pageable": p_w.ctypes.data}
        bl = inputs.blinders
        bad = []

        def submit(jobs, key, pk_, source, ptr, b, link=False):
            c = inputs.circuits[key]
            jobs.append((len(jobs), key, source, b, link, pool.submit_prove(pk_, ptr, c.pub_inputs, bl[b], with_link_poly=link)))

        def collect(jobs, order):
            for i in order:
                j, key, source, b, link, ticket = jobs[i]
                got = pool.wait(ticket)
                proof, poly = got if link else (got, None)
                want, want_poly = refs.proof(key, b)
                if bytes(proof) != want or (link and not (poly == want_poly).all()):
                    bad.append(f"{key} job {j} ({source} wires, blinder set {b}{', link polynomial' if link else ''})")

        # warm-up: three waves of 16, each waited for: every worker proves the key eagerly, captures, replays
        for wave in range(3):
            jobs = []
            for j in range(WORKERS):
                submit(jobs, "synthetic", pk, "device", wires["device"], (wave * WORKERS + j) % N_BLINDERS)
            collect(jobs, range(WORKERS))
        warm_free = torch.cuda.mem_get_info()[0]
        for c in ctxs:
            c.msm_timing_totals(reset=True)
        # 48 proofs, 16 from each kind of memory; blinder set 5 i mod 12: every set 4 times, on whichever workers are free
        jobs = []
        for i, source in enumerate(["device"] * 16 + ["pinned"] * 16 + ["pageable"] * 16):
            submit(jobs, "synthetic", pk, source, wires[source], 5 * i % N_BLINDERS, link=i % 4 == 1)
        collect(jobs, list(range(1, 48, 2))[::-1] + list(range(0, 48, 2)))
        assert not bad, "proofs that differ from the reference bytes: " + "; ".join(bad)
        tot = [c.msm_timing_totals() for c in ctxs]
        assert sum(t["launches"] for t in tot) == 4 * 48
        assert sum(t["pairs"] for t in tot) == 48 * pairs_per_proof(N)
        assert all(math.isfinite(t["accumulate_ms"]) and t["accumulate_ms"] >= 0 for t in tot)
        assert sum(t["accumulate_ms"] for t in tot) > 0
        # the 2^12 private-settlement statement through the same pool, 48 jobs from pinned host memory
        sc = inputs.circuits["settlement"]
        s_bases = ctx.load_bases_device(d_srs.data_ptr(), sc.n + 3)
        s_pk = preprocess(ctx, s_bases, sc)
        s_w = torch.from_numpy(sc.wires.view(np.int64)).pin_memory()
        jobs = []
        for i in range(48):
            submit(jobs, "settlement", s_pk, "pinned", s_w.data_ptr(), i % N_BLINDERS, link=i % 5 == 0)
        collect(jobs, list(range(48))[::-1])
        assert not bad, "proofs that differ from the reference bytes: " + "; ".join(bad)
        # two private-match bundles as bench.py submits them: 5 proofs and 4 link proofs under one ticket each
        circs, link_plan = bundle_circuits
        b_bases = ctx.load_bases_device(d_srs.data_ptr(), (1 << 14) + 3)
        b_pks = [preprocess(ctx, b_bases, c) for c in circs]
        b_w = [torch.from_numpy(c.wires.view(np.int64)).pin_memory() for c in circs]
        tickets = [pool.submit_bundle(b_bases, [(b_pks[j], b_w[j].data_ptr(), circs[j].pub_inputs, bl[(5 * b + j) % N_BLINDERS])
                                                for j in range(5)], [(j, 0, lay) for j, lay in link_plan]) for b in range(2)]
        r_pks = [preprocess(refs.ctx, refs.bases, c) for c in circs]
        for b in (1, 0):
            proofs, polys, links = pool.wait(tickets[b])
            hints = []
            for j, c in enumerate(circs):
                single, hint = PlonkKzgSnark.prove_with_link_hint(refs.ctx, r_pks[j], c.wires, c.pub_inputs, bl[(5 * b + j) % N_BLINDERS])
                assert bytes(proofs[j]) == bytes(single) and (polys[j] == hint.linking_wire_poly).all(), (b, j)
                hints.append(hint)
            for (j, lay), lp in zip(link_plan, links):
                direct, _ = link_proofs(refs.ctx, refs.bases, hints[j], hints[0], lay)
                assert bytes(lp) == bytes(direct), (b, j)
        print(f"pool of {WORKERS} at 2^{LOG_N}: {(free - warm_free) >> 20} MiB of device memory after warm-up "
              f"({free >> 20} MiB free before, {total >> 20} MiB in all)")
        assert pool.stats()["failed"] == 0
        for x in b_pks + r_pks + [s_pk, pk]:
            x.free()
        for x in (b_bases, s_bases, srs):
            x.free()
    finally:
        pool.close()


# ---- MSM timing: bytes unchanged, counts exact -----------------------------------------------------------------------
def check_phases(ph):
    assert all(math.isfinite(v) and v >= 0 for v in ph.values()), ph
    assert ph["total"] > 0 and all(ph["total"] >= ph[k] for k in ("sort", "accumulate", "reduce")), ph


@pytest.mark.parametrize("graphs", [True, False], ids=["graphs", "eager"])
def test_msm_timing_toggled_between_proofs(inputs, refs, graphs):
    """Switching the timing re-captures the prover's graphs (with or without the timing nodes): a stale graph would replay
    without them and leave the phases unrecorded.  The bytes never change; the totals count exactly the proofs made with
    timing on."""
    key = "settlement"
    c = inputs.circuits[key]
    ctx = rb.Context(0)
    ctx.use_graphs(graphs)
    bases = ctx.load_bases(inputs.srs[:c.n + 3])
    pk = preprocess(ctx, bases, c)

    def prove(b):
        proof, hint = PlonkKzgSnark.prove_with_link_hint(ctx, pk, c.wires, c.pub_inputs, inputs.blinders[b])
        want, want_poly = refs.proof(key, b)
        assert bytes(proof) == want and (hint.linking_wire_poly == want_poly).all(), f"blinder set {b}"

    try:
        for b in (0, 1, 2):  # timing off: eager, captured, replayed
            prove(b)
        assert ctx.msm_timing_totals()["launches"] == 0
        ctx.msm_timing(True)
        ctx.msm_timing_totals(reset=True)
        for i, b in enumerate((3, 4, 5)):  # on: re-captured, then replayed
            prove(b)
            check_phases(ctx.msm_timing(True))
            t = ctx.msm_timing_totals()
            assert t["launches"] == 4 * (i + 1) and t["pairs"] == (i + 1) * pairs_per_proof(c.n), t
            assert math.isfinite(t["accumulate_ms"]) and t["accumulate_ms"] > 0
        ctx.msm_timing(False)
        for b in (6, 7):  # off again: re-captured without the timing nodes, nothing counted
            prove(b)
        assert ctx.msm_timing_totals(reset=True)["launches"] == 12
        ctx.msm_timing(True)
        prove(8)
        check_phases(ctx.msm_timing(True))
        t = ctx.msm_timing_totals()
        assert t["launches"] == 4 and t["pairs"] == pairs_per_proof(c.n), t
    finally:
        pk.free()
        bases.free()
        ctx.close()


def test_batch_calls_are_timed_and_counted(inputs, refs, oracle):
    """`prove_batch` and `link_proofs_batch` commit through the context's batch scratch: timing covers it and the totals
    count it — k proofs in 4 launches of 13n + 32 pairs each, k link proofs in 2 launches (quotients, openings)."""
    key = "settlement"
    c = inputs.circuits[key]
    ctx = rb.Context(0)
    bases = ctx.load_bases(inputs.srs[:c.n + 3])
    pk = preprocess(ctx, bases, c)
    try:
        ctx.msm_timing(True)
        ctx.msm_timing_totals(reset=True)
        proofs, _, st = PlonkKzgSnark.prove_batch(ctx, pk, [c.wires] * 3, [c.pub_inputs] * 3, [inputs.blinders[b] for b in (0, 1, 2)])
        assert st == [0, 0, 0]
        for b, p in enumerate(proofs):
            assert bytes(p) == refs.proof(key, b)[0], b
        t = ctx.msm_timing_totals(reset=True)
        assert t["launches"] == 4 and t["pairs"] == 3 * pairs_per_proof(c.n), t
        assert math.isfinite(t["accumulate_ms"]) and t["accumulate_ms"] > 0
        case = ll.BY_NAME["wraps"]
        triples, want = [], []
        for seed in (1, 2):
            h1, h2 = link_hints(oracle, inputs, case, seed)
            triples.append((h1, h2, GroupLayout(case.alignment, case.offset, case.size)))
            want.append(oracle_link(oracle, inputs, case, h1, h2))
        lps, etas, st = link_proofs_batch(ctx, bases, triples)
        assert st == [0, 0]
        for lp, eta, (olp, oeta) in zip(lps, etas, want):
            assert (lp.to_array() == olp.to_array()).all() and (eta == oeta).all()
        t = ctx.msm_timing_totals()
        assert t["launches"] == 2 and t["pairs"] == 2 * case.q_len + 2 * (case.len - 1), t
    finally:
        pk.free()
        bases.free()
        ctx.close()


def link_hints(oracle, inputs, case, seed):
    a1, a2 = ll.pair(oracle, case, seed)
    return [LinkingHint(linking_wire_poly=ll.to_mont(a), linking_wire_comm=oracle.msm(inputs.srs[:len(a)], oracle.ints_to_array(a))[0])
            for a in (a1, a2)]


def oracle_link(oracle, inputs, case, h1, h2):
    rc, olp, oeta = oracle.plonk_link(h1.linking_wire_poly, h2.linking_wire_poly, h1.linking_wire_comm, h2.linking_wire_comm,
                                      case.alignment, case.offset, case.size, inputs.srs[:case.len])
    assert rc == 0
    return olp, oeta


# ---- stream-priority modes ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", [None, "0", "1"], ids=["unset", "0", "1"])
def test_stream_priority_modes(inputs, refs, oracle, monkeypatch, mode):
    """B200_STREAM_PRIORITIES, read by every context at creation: unset, the accumulation and the prover's NTT passes and
    quotient on a low-priority companion stream; 1, the accumulation only; 0, one stream (no companion)."""
    if mode is None:
        monkeypatch.delenv("B200_STREAM_PRIORITIES", raising=False)
    else:
        monkeypatch.setenv("B200_STREAM_PRIORITIES", mode)
    key = "settlement"
    c = inputs.circuits[key]
    bl = inputs.blinders
    ctx = rb.Context(0)
    ctx.use_graphs(True)
    bases = ctx.load_bases(inputs.srs[:c.n + 3])
    pk = preprocess(ctx, bases, c)
    pool = ProverPool(0, workers=4)
    try:
        for b in (0, 1, 2):  # eager, captured, replayed
            proof, _ = PlonkKzgSnark.prove_with_link_hint(ctx, pk, c.wires, c.pub_inputs, bl[b])
            assert bytes(proof) == refs.proof(key, b)[0], f"blinder set {b}"
        for i in range(4):
            pool.context(i).msm_timing(True)
        w = np.ascontiguousarray(c.wires, dtype=np.uint64)
        tickets = [pool.submit_prove(pk, w.ctypes.data, c.pub_inputs, bl[b], keep=w) for b in range(8)]
        for b in reversed(range(8)):
            assert bytes(pool.wait(tickets[b])) == refs.proof(key, b)[0], f"pool job {b}"
        proofs, _, st = PlonkKzgSnark.prove_batch(ctx, pk, [c.wires] * 3, [c.pub_inputs] * 3, [bl[b] for b in (9, 10, 11)])
        assert st == [0, 0, 0]
        for b, p in zip((9, 10, 11), proofs):
            assert bytes(p) == refs.proof(key, b)[0], f"batch item, blinder set {b}"
        case = ll.BY_NAME["len1_far_above_len2"]
        layout = GroupLayout(case.alignment, case.offset, case.size)
        h = [link_hints(oracle, inputs, case, seed) for seed in (3, 4)]
        want = [oracle_link(oracle, inputs, case, *x) for x in h]
        for _ in range(2):  # eager, then captured
            lp, eta = link_proofs(ctx, bases, h[0][0], h[0][1], layout)
            assert (lp.to_array() == want[0][0].to_array()).all() and (eta == want[0][1]).all()
        lps, etas, st = link_proofs_batch(ctx, bases, [(x[0], x[1], layout) for x in h])
        assert st == [0, 0]
        for lp, eta, (olp, oeta) in zip(lps, etas, want):
            assert (lp.to_array() == olp.to_array()).all() and (eta == oeta).all()
        n = 1 << 12
        for wb in (1, 0):  # a lone latency-plan MSM, a lone throughput-plan MSM
            mb = ctx.load_bases(inputs.srs[:n], window_bits=wb)
            out, inf = ctx.msm(mb, inputs.scalars[:n])
            exp, einf = oracle.msm(inputs.srs[:n], inputs.scalars[:n])
            assert inf == einf and (out == exp).all(), f"window_bits={wb}"
            mb.free()
    finally:
        pool.close()
        pk.free()
        bases.free()
        ctx.close()


# ---- process-wide switches, one subprocess each ---------------------------------------------------------------------------
@pytest.fixture(scope="module")
def driver_inputs(inputs, tmp_path_factory):
    path = tmp_path_factory.mktemp("regime") / "inputs.npz"
    arrays = {"srs": inputs.srs, "blinders": inputs.blinders, "scalars": inputs.scalars, "batch_scalars": inputs.batch_scalars,
              "seed_srs": np.array(SEED_SRS)}
    for name, vals in inputs.one_base.items():
        arrays[f"one_base_{name}"] = np.stack([np.array([(v >> (64 * k)) & (2**64 - 1) for k in range(4)], dtype=np.uint64)
                                               for v in vals])
    for key, c in inputs.circuits.items():
        for f in ("selectors", "perm", "k", "wires", "pub_inputs"):
            arrays[f"{key}_{f}"] = np.ascontiguousarray(getattr(c, f))
    np.savez(path, **arrays)
    return path


@pytest.fixture(scope="module")
def msm_expected(inputs, oracle):
    """What the driver's MSMs must return, from the oracle"""
    srs, s = inputs.srs, inputs.scalars
    exp = {}
    for lg in (12, 14, 16):
        exp[f"latency_2^{lg}"] = oracle.msm(srs[:1 << lg], s[:1 << lg])
    exp["throughput_2^16"] = exp["latency_2^16"]
    one = np.repeat(srs[:1], 256, axis=0)
    for name, vals in inputs.one_base.items():
        for wb in (1, 0):
            exp[f"one_base_{name}_w{wb}"] = oracle.msm(one, oracle.ints_to_array(vals))
    for b in (5, 12):
        exp[f"batch_{b}"] = [oracle.msm(srs[:1 << 12], inputs.batch_scalars[i]) for i in range(b)]
    return exp


def run_driver(path, mode, env_set):
    env = {k: v for k, v in os.environ.items() if k not in SWITCHES}
    env.update(env_set)
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + [DRIVER, str(path), mode]
    r = subprocess.run(cmd, env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, f"{env_set}: exit {r.returncode}\n{r.stderr[-3000:]}"
    return json.loads(r.stdout.strip().splitlines()[-1])


def check_proofs(got, refs, label):
    bad = [f"{key} #{i} (blinder set {b})" for key, items in got.items() for i, (b, hx) in enumerate(items)
           if bytes.fromhex(hx) != refs.proof(key.replace("_batch", ""), b)[0]]
    assert not bad, f"{label}: proofs that differ from the reference bytes: " + "; ".join(bad)


SETTINGS = [{"B200_QUAD_ADD": "0"}, {"B200_QUAD_ADD": "1"}, {"B200_TREE_FANIN_LOG": "1"}, {"B200_TREE_FANIN_LOG": "2"},
            {"B200_TREE_FANIN_LOG": "3"}, {"B200_HOST_HORNER": "0"}, {"B200_GRAPHS": "0"}]


@pytest.mark.parametrize("setting", SETTINGS, ids=["-".join(f"{k}={v}" for k, v in s.items()) for s in SETTINGS])
def test_process_wide_switch(driver_inputs, msm_expected, refs, setting):
    got = run_driver(driver_inputs, "switches", setting)
    label = ", ".join(f"{k}={v}" for k, v in setting.items())
    bad = []
    for name, exp in msm_expected.items():
        items = got["msm"][name] if isinstance(exp, list) else [got["msm"][name]]
        for i, ((xy, inf), (ex, einf)) in enumerate(zip(items, exp if isinstance(exp, list) else [exp])):
            if inf != einf or np.frombuffer(bytes.fromhex(xy), dtype=np.uint64).tolist() != ex.tolist():
                bad.append(f"{name}[{i}]")
    assert not bad, f"{label}: MSMs that differ from the oracle: {bad}"
    assert got["batch_statuses"] == [0, 0]
    check_proofs(got["proofs"], refs, label)
    # the MSMs reached the shapes they are here for (default B200_TREE_FANIN_LOG / B200_QUAD_ADD): a fan-in-4 serial tree
    # level for the lone latency plans (four lanes per addition at 2^12); the batch of 12 crosses to fan-in 8
    forced = int(setting.get("B200_TREE_FANIN_LOG", 0))
    plans = got["plans"]
    for lg in (12, 14, 16):
        assert plans[f"latency_2^{lg}"]["window_bits"] >= 5
        a_row, a_col, quad = serial_level(plans[f"latency_2^{lg}"], forced=forced)
        if not forced:
            assert (a_row, a_col) == (2, 2), (lg, plans[f"latency_2^{lg}"])
            assert quad == (lg == 12), (lg, plans[f"latency_2^{lg}"])
    if not forced:
        assert serial_level(plans["batch"], batch=5)[:2] == (2, 2) and serial_level(plans["batch"], batch=12)[:2] == (3, 3)


def test_bench_environment_pool_of_16(driver_inputs, refs):
    """bench.py's process: CUDA_DEVICE_MAX_CONNECTIONS=32 before CUDA starts, a pool of 16 at 2^16 with timing on, SRS made
    and loaded on the device; 48 proofs from device memory, 16 from pinned host memory."""
    import torch
    free, total = torch.cuda.mem_get_info()
    if free < POOL_BYTES:
        pytest.skip(f"a pool of {WORKERS} at 2^{LOG_N} wants {POOL_BYTES >> 20} MiB free, the GPU has {free >> 20} of "
                    f"{total >> 20} MiB free")
    got = run_driver(driver_inputs, "pool16", {"CUDA_DEVICE_MAX_CONNECTIONS": "32"})
    assert got["cuda_device_max_connections"] == "32"
    check_proofs(got["proofs"], refs, "CUDA_DEVICE_MAX_CONNECTIONS=32, pool of 16")
    assert got["msm_launches"] == 4 * 64
