"""GPU: compact proving keys (include/b200compact.h) give the default key's bytes through every prover entry point, and
make 2^23 provable on one 80 GB H100.

- The verifying key of a compact key = the default key's at every n = 2^2 … 2^17, from the permutation and from the
  wiring; proofs = the default key's (every commitment, evaluation, challenge and the linking polynomial) at every
  n = 2^2 … 2^17 and at 2^20, eagerly and from replayed graphs, across 8 cosets (n < 16) and 6.
- prove_witness, prove_batch of 1, 3 and 17, a settlement with four hints, and the pool's single, bundle and batch jobs
  on compact keys = the default key's bytes.
- A default and a compact key of one circuit interleaved on one context keep their own graphs: correct bytes after
  every switch.
- Every case of `unsat_shapes.catalogue` at 2^10 and the low-degree cases at 2^16 are refused with B200_ERR_UNSATISFIED
  exactly where the default key refuses them, each followed by a control proof (the case's satisfying witness, with
  blinders of its own) with the default key's bytes.
- 2^23 on a context of its own (skipped, with the numbers, when free memory is below the compact estimate × 1.15):
  two proofs, one eager and one replayed, with other blinders, from the table and from the witness, each accepted by
  the oracle's known-τ verifier and the three device verifiers; a flipped evaluation bit and a changed public input
  rejected by all four; a gate violation refused and the next honest proof unchanged; device memory within the
  estimate."""
import gc
import time

import numpy as np
import pytest
import torch

import large_domains as ld
import unsat_shapes as us
import renegade_b200 as rb
from renegade_b200 import _lib, synth
from renegade_b200.backend import B200Proof, GroupLayout, PlonkKzgSnark, ProverPool, VerifyingKey

pytestmark = pytest.mark.gpu

TAU = 0x2C0FFEE0B5E55ED1A2B3C4D5E6F708192A3B4C5D6E7F8091A2B3C4D5E6F70819
SLACK = 1.15
UNSAT = _lib.B200_ERR_UNSATISFIED


def _tau(oracle, pyoracle):
    return oracle.int_to_limbs(pyoracle.to_mont(TAU % pyoracle.R, pyoracle.R))


@pytest.fixture(scope="module")
def srs17(oracle, pyoracle):
    """(τ, the first 2^17 + 3 powers of τ): every size up to 2^17 loads its own n + 3 of them"""
    tau = _tau(oracle, pyoracle)
    return tau, oracle.srs_from_tau(tau, (1 << 17) + 3)


@pytest.fixture(scope="module")
def cctx():
    c = rb.Context(0)
    yield c
    c.close()


def _circuit(log_n, seed=0xC0):
    return synth.synth_circuit(log_n, num_inputs=1 if log_n < 4 else 3, seed=seed + log_n)


class Keys:
    """One circuit's default and compact keys, from the permutation and from the wiring, on one context."""

    def __init__(self, ctx, srs, log_n, circ=None, wiring=True):
        self.ctx, self.log_n = ctx, log_n
        self.c = c = circ or _circuit(log_n)
        self.bases = ctx.load_bases(srs[:(1 << log_n) + 3])
        self.pk = PlonkKzgSnark.preprocess(ctx, self.bases, log_n, c.num_inputs, c.selectors, c.perm, c.k)
        self.cpk = PlonkKzgSnark.preprocess(ctx, self.bases, log_n, c.num_inputs, c.selectors, c.perm, c.k, compact=True)
        self.wpk = self.cwpk = None
        if wiring:
            args = (ctx, self.bases, log_n, c.num_inputs, c.selectors, c.wire_vars, len(c.witness), c.k)
            self.wpk = PlonkKzgSnark.preprocess_wiring(*args)
            self.cwpk = PlonkKzgSnark.preprocess_wiring(*args, compact=True)

    def prove(self, pk, bl):
        """(proof bytes, link polynomial, challenges)"""
        p, h, ch = PlonkKzgSnark.prove_with_link_hint(self.ctx, pk, self.c.wires, self.c.pub_inputs, bl, want_challenges=True)
        return bytes(p), h.linking_wire_poly.copy(), ch.copy()

    def free(self):
        for k in (self.pk, self.cpk, self.wpk, self.cwpk, self.bases):
            if k is not None:
                k.free()


def same_vk(a, b):
    return (a.selector_comms == b.selector_comms).all() and (a.sigma_comms == b.sigma_comms).all()


def same(x, y):
    return x[0] == y[0] and (x[1] == y[1]).all() and (x[2] == y[2]).all()


def check_size(ctx, srs, log_n):
    ks = Keys(ctx, srs, log_n)
    try:
        assert ks.cpk.compact and ks.cwpk.compact and not ks.pk.compact and not ks.wpk.compact
        # (synth's permutation is not the one the wiring derives: the wiring keys are compared with each other)
        assert same_vk(ks.pk, ks.cpk) and same_vk(ks.wpk, ks.cwpk), log_n
        bl = synth.splitmix_blinders(0xC1 + log_n)
        ref = ks.prove(ks.pk, bl)
        assert same(ks.prove(ks.cpk, bl), ref), f"2^{log_n}: compact eager"
        g0 = ctx.graph_launches()
        for i in range(2):  # captured, then replayed
            assert same(ks.prove(ks.cpk, bl), ref), f"2^{log_n}: compact graphs, call {i}"
        assert ctx.graph_launches() - g0 == 2 * 6  # a default key replays 7 segments a proof, a compact one 6: no side stream
        bl2 = synth.splitmix_blinders(0xC2 + log_n)
        assert same(ks.prove(ks.cpk, bl2), ks.prove(ks.pk, bl2)), f"2^{log_n}: other blinders"
        wref = PlonkKzgSnark.prove_witness(ctx, ks.wpk, ks.c.witness, bl, want_challenges=True)
        for _ in range(3):  # eager, captured, replayed
            wp, wh, wpub, wch = PlonkKzgSnark.prove_witness(ctx, ks.cwpk, ks.c.witness, bl, want_challenges=True)
            assert bytes(wp) == bytes(wref[0]) and (wh.linking_wire_poly == wref[1].linking_wire_poly).all()
            assert (wpub == ks.c.pub_inputs).all() and (wch == wref[3]).all()
    finally:
        ks.free()


@pytest.mark.parametrize("log_n", range(2, 18))
def test_keys_and_proofs_equal_the_default_keys(cctx, srs17, log_n):
    check_size(cctx, srs17[1], log_n)


def test_2_20_proofs_equal_the_default_keys(oracle, pyoracle):
    tau = _tau(oracle, pyoracle)
    srs = oracle.srs_from_tau(tau, (1 << 20) + 3)
    ctx = rb.Context(0)
    try:
        check_size(ctx, srs, 20)
    finally:
        ctx.close()


@pytest.mark.parametrize("log_n", [3, 10])
def test_batches_and_settlements(cctx, srs17, log_n):
    """prove_batch of 1, 3 and 17 on the compact key = single proofs of the default key; a settlement with four hints
    (the statement's own circuit proved with other blinders, over four layouts) = the default key's settlement."""
    ks = Keys(cctx, srs17[1], log_n, wiring=False)
    try:
        c, n = ks.c, 1 << log_n
        bls = [synth.splitmix_blinders(0xD0 + i) for i in range(17)]
        singles = {i: ks.prove(ks.pk, bls[i]) for i in range(17)}
        for k in (1, 3, 17):
            proofs, hints, st = PlonkKzgSnark.prove_batch(cctx, ks.cpk, [c.wires] * k, [c.pub_inputs] * k, bls[:k],
                                                          link_hints=True)
            assert list(st) == [0] * k
            for i in range(k):
                assert bytes(proofs[i]) == singles[i][0] and (hints[i].linking_wire_poly == singles[i][1]).all(), (k, i)
        _, hint, _ = PlonkKzgSnark.prove_with_link_hint(cctx, ks.pk, c.wires, c.pub_inputs, bls[5], want_challenges=True)
        layouts = [GroupLayout(log_n, 1, 2), GroupLayout(log_n, n // 2, n // 4), GroupLayout(2, 0, 4), GroupLayout(log_n, n - 3, 3)]
        links = [(hint, lay) for lay in layouts]
        out = {}
        for name, pk in (("default", ks.pk), ("compact", ks.cpk)):
            proof, lps, st = PlonkKzgSnark.prove_settlement(cctx, ks.bases, pk, c.wires, c.pub_inputs, bls[0], links)
            assert list(st) == [0] * 5, name
            out[name] = (bytes(proof), [bytes(lp) for lp in lps])
        assert out["compact"] == out["default"] and out["default"][0] == singles[0][0]
    finally:
        ks.free()


def test_pool_jobs(srs17):
    """A pool of two workers: a single witness job, a bundle of two witness proofs and a link, and a batch job of three
    on compact keys = the same jobs on the default keys."""
    pool = ProverPool(0, workers=2)
    try:
        ctx = pool.context(0)
        ks = Keys(ctx, srs17[1], 12)
        c = ks.c
        bl = [synth.splitmix_blinders(0xE0 + i) for i in range(3)]
        layout = GroupLayout(12, 100, 16)
        res = {}
        for name, pk, wpk in (("default", ks.pk, ks.wpk), ("compact", ks.cpk, ks.cwpk)):
            single = pool.wait(pool.submit_prove_witness(wpk, c.witness, bl[0]))
            bundle = pool.wait(pool.submit_bundle_witness(ks.bases, [(wpk, c.witness, bl[0]), (wpk, c.witness, bl[1])],
                                                          [(0, 1, layout)]))
            proofs, _, st = pool.wait(pool.submit_prove_batch(pk, [c.wires] * 3, [c.pub_inputs] * 3, bl))
            assert list(st) == [0] * 3
            res[name] = (bytes(single[0]), [bytes(p) for p in bundle[0]], [bytes(lp) for lp in bundle[2]],
                         [bytes(p) for p in proofs])
        assert res["compact"] == res["default"]
        assert res["default"][0] == res["default"][1][0]
        ks.free()
    finally:
        pool.close()


def test_default_and_compact_keys_interleaved(cctx, srs17):
    """Proofs alternate between the two keys of one circuit on one context: each key captures its own graphs on its
    second proof and replays them afterwards, and every proof has the reference bytes."""
    ks = Keys(cctx, srs17[1], 11, wiring=False)
    try:
        bl = synth.splitmix_blinders(0xF1)
        ref = ks.prove(ks.pk, bl)
        for i in range(3):
            for pk in (ks.cpk, ks.pk, ks.cpk):
                g0 = cctx.graph_launches()
                assert same(ks.prove(pk, bl), ref), (i, pk.compact)
                if i:  # every key has run eagerly and captured by now
                    assert cctx.graph_launches() - g0 == (6 if pk.compact else 7)
    finally:
        ks.free()


def _unsat_cases():
    return us.catalogue(10) + [us.low_degree(16, p) for p in us.LOW_DEGREE]


def test_unsatisfied_refused_where_the_default_key_refuses(cctx, oracle, pyoracle):
    """Each case's witness on the default and the compact key: the same status (B200_ERR_UNSATISFIED, or the same
    proof bytes), then a control proof of the case's satisfying witness on the compact key = the default key's."""
    tau = _tau(oracle, pyoracle)
    srs = oracle.srs_from_tau(tau, (1 << 16) + 3)
    seen = {"refused": 0, "proved": 0}
    cbl = synth.splitmix_blinders(0xC7)
    for case in _unsat_cases():
        sel, wires, pub, perm, k, bl = case.tables()
        bases = cctx.load_bases(srs[:case.n + 3])
        pk = PlonkKzgSnark.preprocess(cctx, bases, case.log_n, case.num_inputs, sel, perm, k)
        cpk = PlonkKzgSnark.preprocess(cctx, bases, case.log_n, case.num_inputs, sel, perm, k, compact=True)
        good_wires, good_pub = case.good
        gw = np.stack([synth.to_mont_array(col) for col in good_wires])
        gp = synth.to_mont_array(good_pub).reshape(-1, 4)

        def attempt(key, w, p, b=bl):
            try:
                return 0, bytes(PlonkKzgSnark.prove_with_link_hint(cctx, key, w, p, b)[0])
            except _lib.B200Error as e:
                assert e.code == UNSAT and "WrongQuotientPolyDegree" in str(e), (case.name, e)
                return UNSAT, None

        try:
            for _ in range(2):  # the keys' first, eager calls; then captured graphs
                got = attempt(cpk, wires, pub)
                assert got == attempt(pk, wires, pub), case.name
                assert got[0] == (UNSAT if case.expect == us.UNSAT else 0), case.name
                control = attempt(cpk, gw, gp, cbl)  # blinders of its own: a blinder case's are refused by design
                assert control == attempt(pk, gw, gp, cbl) and control[0] == 0, case.name
            seen["refused" if got[0] else "proved"] += 1
        finally:
            for h in (pk, cpk, bases):
                h.free()
    print(f"unsatisfied catalogue on compact keys: {seen}")
    assert seen["refused"] > 40


# ---- 2^23 ---------------------------------------------------------------------------------------------------------
def _free():
    gc.collect()
    torch.cuda.empty_cache()
    return torch.cuda.mem_get_info()


def test_2_23_on_one_gpu(oracle, pyoracle, g2_raw):
    import bn254_pairing_py as pr
    log_n, n = 23, 1 << 23
    parts = PlonkKzgSnark.footprint(log_n, 1, compact=True)
    est = sum(parts.values())
    free, total = _free()
    print(f"\n2^23 compact: estimate {est / 2**30:.2f} GiB ({', '.join(f'{k} {v / 2**30:.2f}' for k, v in parts.items() if v)}), "
          f"{free / 2**30:.2f} of {total / 2**30:.2f} GiB free", flush=True)
    if free < est * SLACK:
        pytest.skip(f"2^23: {int(est * SLACK) >> 20} MiB wanted (compact estimate x {SLACK}), {free >> 20} of {total >> 20} MiB free")
    t0 = time.time()
    circ = ld.big_circuit(log_n, seed=0x23)
    tau = _tau(oracle, pyoracle)
    srs = oracle.srs_from_tau(tau, n + 3)
    h = g2_raw[0]
    tau_h = np.frombuffer(pr.encode_g2_mont(pr.g2_mul(pr.decode_g2_mont(h.tobytes(), 0), TAU % pr.R)), dtype=np.uint64).copy()
    print(f"2^23: circuit and SRS on the host in {time.time() - t0:.1f} s", flush=True)
    free0 = _free()[0]
    ctx = rb.Context(0)
    peak = 0

    def measure(what):
        nonlocal peak
        used = free0 - torch.cuda.mem_get_info()[0]
        peak = max(peak, used)
        print(f"2^23 {what}: {used / 2**30:.2f} GiB in use on the device (estimate {est / 2**30:.2f})", flush=True)

    def verdicts(pk, pub, proof):
        opk = {"selector_comms": pk.selector_comms, "sigma_comms": pk.sigma_comms}
        vk = VerifyingKey.from_proving_key(pk, h, tau_h)
        ok_b, v_b = PlonkKzgSnark.batch_verify(ctx, [vk], [pub], [proof])
        return (oracle.plonk_verify_known_tau(log_n, circ.num_inputs, circ.k, opk, pub,
                                              oracle.PlonkProof.from_buffer_copy(bytes(proof)), tau),
                PlonkKzgSnark.verify(vk, pub, proof), ok_b and v_b == [True],
                PlonkKzgSnark.verify_each(ctx, [vk], [pub], [proof]) == [True])

    try:
        bases = ctx.load_bases(srs)
        del srs
        t0 = time.time()
        pk = PlonkKzgSnark.preprocess(ctx, bases, log_n, circ.num_inputs, circ.selectors, circ.perm, circ.k, compact=True)
        print(f"2^23: compact key in {time.time() - t0:.1f} s", flush=True)
        measure("compact key")
        bl, bl2 = synth.splitmix_blinders(0x2301), synth.splitmix_blinders(0x2302)
        times = []
        proofs = []
        for b in (bl, bl2, bl2):  # eager; captured; replayed
            t0 = time.time()
            proofs.append(PlonkKzgSnark.prove_with_link_hint(ctx, pk, circ.wires, circ.pub_inputs, b)[0])
            times.append(time.time() - t0)
        print(f"2^23: proofs in {', '.join(f'{t:.2f}' for t in times)} s (eager, captured, replayed)", flush=True)
        measure("key and three proofs")
        assert bytes(proofs[1]) == bytes(proofs[2]) != bytes(proofs[0])
        for p in (proofs[0], proofs[2]):
            assert verdicts(pk, circ.pub_inputs, p) == (True,) * 4
        bad = B200Proof.from_buffer_copy(bytes(proofs[2]))
        bad.wires_evals[2][0] ^= 1
        assert verdicts(pk, circ.pub_inputs, bad) == (False,) * 4
        wrong = circ.pub_inputs.copy()
        wrong[-1] = circ.pub_inputs[0] if (circ.pub_inputs[0] != circ.pub_inputs[-1]).any() else circ.pub_inputs[1]
        assert verdicts(pk, wrong, proofs[2]) == (False,) * 4
        # a gate violation, refused from the replayed graphs; the next honest proof is unchanged
        wv = circ.wire_vars
        counts = np.bincount(wv.reshape(-1))
        row = next(r for r in sorted(circ.gate_rows) if r > n // 2 and circ.gate_rows[r] == "hash")
        col = next(i for i in (1, 2, 3) if counts[wv[i, row]] == 1)
        gate_bad = circ.wires.copy()
        gate_bad[col, row] = ld.random_fr(np.random.default_rng(1), 1)[0]
        with pytest.raises(_lib.B200Error) as ei:
            PlonkKzgSnark.prove_with_link_hint(ctx, pk, gate_bad, circ.pub_inputs, bl2)
        assert ei.value.code == UNSAT
        assert bytes(PlonkKzgSnark.prove_with_link_hint(ctx, pk, circ.wires, circ.pub_inputs, bl2)[0]) == bytes(proofs[2])
        ref = bytes(proofs[0])
        del proofs, bad
        pk.free()
        # from the wiring and the witness vector: the same bytes
        wpk = PlonkKzgSnark.preprocess_wiring(ctx, bases, log_n, circ.num_inputs, circ.selectors, circ.wire_vars,
                                              circ.num_vars, circ.k, compact=True)
        assert same_vk(wpk, pk)
        wproof, _, wpub = PlonkKzgSnark.prove_witness(ctx, wpk, circ.witness, bl)
        assert bytes(wproof) == ref and (wpub == circ.pub_inputs).all()
        assert verdicts(wpk, circ.pub_inputs, wproof) == (True,) * 4
        measure("wiring key and its proof")
        wpk.free()
        bases.free()
    finally:
        ctx.close()
    print(f"2^23: peak {peak / 2**30:.2f} GiB measured, estimate {est / 2**30:.2f} GiB", flush=True)
    assert peak <= est
