"""Verification jobs (`ProverPool.submit_verify`) beside proof traffic, against the path a caller without them takes:
verifying on a bare context of its own beside the pool.

    python tools/verify_jobs_bench.py [--proofs 960] [--repeats 3]

One pool of 16 workers proves the PRIVATE SETTLEMENT (2^12) and OUTPUT BALANCE VALIDITY (2^13) statements of a private
match (examples/host_circuits), alternating, from witness vectors, `--proofs` proofs per window with 16 in flight.  At the
same time one host thread sends a stream of gossip-shaped verification jobs, one after the other: k orders per job, each
order two proofs (the validity proof and the settlement proof) and their link proof, k = 1, 16, 256.  Paths:
  none          no verification stream (proof traffic alone)
  pool-each     submit_verify on the same pool, per-item mode (b200_plonk_verify_each on a worker's context)
  pool-comb     submit_verify(combined=True) on the same pool (b200_plonk_batch_verify on a worker's context)
  ctx-each      PlonkKzgSnark.verify_each on a separate bare context beside the pool (the caller's path today)
  ctx-comb      PlonkKzgSnark.batch_verify on that context
Per window it reports proofs/s and the verdict latency of every verification job (submit to verdicts in hand), median
(min, max); the windows of every path and k alternate, `--repeats` rounds.  Every verdict is checked to be true, and the
pool's verdicts equal the bare context's.  Also the device memory, from the free memory the driver reports: what the
process's first verifications (pool jobs, every k, both modes) take, then what one extra context adds on top, after
`b200_init` and after its own verifications.  Clocks and power limit are used as found; the first line names
the card, its power limit and maximum SM clock.  One JSON line per result.
"""
import argparse
import json
import os
import sys
import threading
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "examples"))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

import numpy as np  # noqa: E402

from bundle_witness_bench import card, private_match, spread  # noqa: E402

TAU = 0x7A0C1D2E3F405162738495A6B7C8D9E0F1021324354657687980A1B2C3D4E5F6  # of the seeded SRS the proofs are made on
KS = (1, 16, 256)
PATHS = ("pool-each", "pool-comb", "ctx-each", "ctx-comb")


def seeded_srs(n):
    """n powers tau^i G (the oracle's C restatement) and the G2 pair (h, tau h) a verifier needs for them."""
    import bn254_pairing_py as pr
    import bn254_py as py
    import oracle_c
    oracle_c.build()
    pts = oracle_c.srs_from_tau(oracle_c.int_to_limbs(py.to_mont(TAU % py.R, py.R)), n)
    with open(os.path.join(ROOT, "tests", "golden", "srs_g2.bin"), "rb") as f:
        h = np.frombuffer(f.read(128), dtype=np.uint64).copy()
    tau_h = np.frombuffer(pr.encode_g2_mont(pr.g2_mul(pr.decode_g2_mont(h.tobytes(), 0), TAU % pr.R)), dtype=np.uint64).copy()
    return pts, h, tau_h


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--proofs", type=int, default=960)
    ap.add_argument("--repeats", type=int, default=3)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("verify_jobs_bench: no CUDA device (there is nothing to measure without one)")
    import renegade_b200 as rb
    from renegade_b200 import synth
    from renegade_b200.backend import PlonkKzgSnark, ProverPool, VerifyingKey, link_proofs

    name, power = card()
    print(json.dumps({"card": name, "power_limit,max_sm_clock": power}), flush=True)
    circs, links = private_match()
    sel = [0, 3]  # PRIVATE SETTLEMENT (2^12), OUTPUT BALANCE VALIDITY (2^13) of party 0
    (a, b, lay), = [(a, b, lay) for a, b, lay in links if a == 3]
    pool = ProverPool(0, workers=16)
    pc = pool.context(0)
    pts, h, tau_h = seeded_srs(max(circs[j].n for j in sel) + 3)
    bases = pc.load_bases(pts)
    pks = {j: PlonkKzgSnark.preprocess_wiring(pc, bases, circs[j].log_n, circs[j].num_inputs, circs[j].selectors,
                                              circs[j].wire_vars, circs[j].num_vars, circs[j].k) for j in sel}
    wits = {j: np.ascontiguousarray(circs[j].witness) for j in sel}
    bl = [synth.splitmix_blinders(9100 + i) for i in range(8)]
    made = {j: PlonkKzgSnark.prove_witness(pc, pks[j], wits[j], bl[j]) for j in sel}  # (proof, hint, pub)
    vks = {j: VerifyingKey.from_proving_key(pks[j], h, tau_h) for j in sel}
    lp, _ = link_proofs(pc, bases, made[a][1], made[b][1], lay)
    order_proofs = [(vks[a], made[a][2], made[a][0]), (vks[b], made[b][2], made[b][0])]
    order_link = (made[a][1].linking_wire_comm, made[b][1].linking_wire_comm, lp, lay)

    def items(k):
        ps = order_proofs * k
        return [p[0] for p in ps], [p[1] for p in ps], [p[2] for p in ps], [order_link] * k

    jobs = {k: items(k) for k in KS}
    # device memory: the process's first verifications (on the pool), then what one more context adds on top
    free0, _ = torch.cuda.mem_get_info(0)
    first = {k: pool.wait(pool.submit_verify(*jobs[k], g2=(h, tau_h))) for k in KS}
    for k in KS:
        pool.wait(pool.submit_verify(*jobs[k], combined=True, g2=(h, tau_h)))
    free1, _ = torch.cuda.mem_get_info(0)
    ctx = rb.Context(0)  # the bare context a caller keeps today
    free2, _ = torch.cuda.mem_get_info(0)
    want = {k: PlonkKzgSnark.verify_each(ctx, *jobs[k], g2=(h, tau_h)) for k in KS}
    for k in KS:
        PlonkKzgSnark.batch_verify(ctx, *jobs[k], g2=(h, tau_h))
    free3, _ = torch.cuda.mem_get_info(0)
    assert all(all(w) for w in want.values()) and first == want
    print(json.dumps({"device_bytes": {"first_verifications_in_the_process": int(free0 - free1),
                                       "extra_context_after_b200_init": int(free1 - free2),
                                       "extra_context_after_its_verifications": int(free1 - free3)}}), flush=True)

    def verify(path, k):
        if path == "pool-each":
            return pool.wait(pool.submit_verify(*jobs[k], g2=(h, tau_h)))
        if path == "pool-comb":
            ok, v = pool.wait(pool.submit_verify(*jobs[k], combined=True, g2=(h, tau_h)))
            assert ok
            return v
        if path == "ctx-each":
            return PlonkKzgSnark.verify_each(ctx, *jobs[k], g2=(h, tau_h))
        ok, v = PlonkKzgSnark.batch_verify(ctx, *jobs[k], g2=(h, tau_h))
        assert ok
        return v

    def window(path, k):
        """--proofs proofs with 16 in flight; the verification stream runs until the last proof is in."""
        done, lat = threading.Event(), []

        def stream():
            while not done.is_set():
                t = time.perf_counter()
                v = verify(path, k)
                lat.append((time.perf_counter() - t) * 1e3)
                assert v == want[k], (path, k)

        th = threading.Thread(target=stream) if path != "none" else None
        t0 = time.perf_counter()
        if th:
            th.start()
        inflight, i = [], 0
        while i < args.proofs or inflight:
            while i < args.proofs and len(inflight) < 16:
                j = sel[i % 2]
                inflight.append(pool.submit_prove_witness(pks[j], wits[j], bl[i % 8]))
                i += 1
            pool.wait(inflight.pop(0))
        rate = args.proofs / (time.perf_counter() - t0)
        done.set()
        if th:
            th.join()
        return rate, lat

    # warm-up: every worker has proved both keys (graphs captured) and every path has run every k
    window("none", 1)
    for path in PATHS:
        for k in KS:
            verify(path, k)
    rates = {("none", 0): []}
    lats = {}
    for _ in range(args.repeats):
        r, _ = window("none", 0)
        rates[("none", 0)].append(r)
        for k in KS:
            for path in PATHS:
                r, lat = window(path, k)
                rates.setdefault((path, k), []).append(r)
                lats.setdefault((path, k), []).extend(lat)
    print(json.dumps({"path": "none", "proofs_per_s": spread(rates[("none", 0)])}), flush=True)
    for k in KS:
        for path in PATHS:
            print(json.dumps({"path": path, "orders_per_job": k, "items_per_job": 3 * k,
                              "proofs_per_s": spread(rates[(path, k)]), "verdict_ms": spread(lats[(path, k)]),
                              "jobs": len(lats[(path, k)])}), flush=True)
    ctx.close()
    for pk in pks.values():
        pk.free()
    bases.free()
    pool.close()


if __name__ == "__main__":
    main()
