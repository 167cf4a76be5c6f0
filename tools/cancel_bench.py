"""Cancellation (include/b200cancel.h) on the GPU: how long a pool takes to stop, and what the abort points cost a proof.

    python tools/cancel_bench.py [--queued 256] [--verify-k 4096] [--proofs 200]

1. Stop time.  A pool of 4 workers gets a deep queue of `--queued` proofs of one synthetic circuit (2^12, 2^13 and 2^16 in
   turn), or one combined verification job over `--verify-k` items with every other item tampered (its bisection runs
   for tens of seconds).  As soon as the work has started, the pool is stopped either with `b200_pool_destroy` alone (it
   drains the queue) or with `cancel_all` then `destroy`; the time from that call to the destroy's return is reported for
   both, with the number of jobs `cancel_all` dropped.
2. Check cost.  The same proof (2^13) made `--proofs` times one after the other on a pool worker, whose calls test the
   cancel flag at every abort point and never find it set, and on a bare context, whose calls have no flag; median and
   p10 / p90 of each, and their difference.  The worker's time also holds the pool's queue hand-off.

The first line names the card, its power limit and maximum SM clock, read in the same run.  One JSON line per result.
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

import numpy as np  # noqa: E402

from bundle_witness_bench import card  # noqa: E402
from verify_jobs_bench import seeded_srs  # noqa: E402


def percentiles(xs):
    a = np.asarray(xs, dtype=np.float64) * 1e3
    return {"median_ms": float(np.median(a)), "p10_ms": float(np.percentile(a, 10)), "p90_ms": float(np.percentile(a, 90))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--queued", type=int, default=256)
    ap.add_argument("--verify-k", type=int, default=4096)
    ap.add_argument("--proofs", type=int, default=200)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("cancel_bench: no CUDA device (there is nothing to measure without one)")
    import renegade_b200 as rb
    from renegade_b200 import synth
    from renegade_b200.backend import B200Proof, PlonkKzgSnark, ProverPool, VerifyingKey

    name, power = card()
    print(json.dumps({"card": name, "power_limit,max_sm_clock": power}), flush=True)
    ctx = rb.Context(0)
    pts, h, tau_h = seeded_srs((1 << 16) + 3)
    bases = ctx.load_bases(pts)
    keys = {}
    for log_n in (12, 13, 16):
        c = synth.synth_circuit(log_n, num_inputs=2, seed=9500 + log_n)
        pk = PlonkKzgSnark.preprocess_wiring(ctx, bases, c.log_n, c.num_inputs, c.selectors, c.wire_vars, c.num_vars, c.k)
        keys[log_n] = (c, pk)

    def stop(fill, cancel):
        pool = ProverPool(0, workers=4)
        tickets = fill(pool)
        while pool.stats()["queued"] >= len(tickets):
            time.sleep(0.0005)  # until work has started
        t0 = time.perf_counter()
        dropped = pool.cancel_all() if cancel else 0
        pool.close()
        return time.perf_counter() - t0, dropped, len(tickets)

    def proofs(log_n):
        c, pk = keys[log_n]
        bl = synth.splitmix_blinders(9600)
        return lambda pool: [pool.submit_prove_witness(pk, c.witness, bl) for _ in range(args.queued)]

    c13, pk13 = keys[13]
    p13, _, pub13 = PlonkKzgSnark.prove_witness(ctx, pk13, c13.witness, synth.splitmix_blinders(9601))
    vk13 = VerifyingKey.from_proving_key(pk13, h, tau_h)
    bad = B200Proof.from_buffer_copy(p13)
    bad.wires_evals[0][0] ^= 1
    k = args.verify_k
    vargs = ([vk13] * k, [pub13] * k, [p13 if i % 2 == 0 else bad for i in range(k)])

    def verify(pool):
        return [pool.submit_verify(*vargs, combined=True, g2=(h, tau_h))]

    cases = [(f"{args.queued} proofs of 2^{n} queued", proofs(n)) for n in (12, 13, 16)]
    cases.append((f"combined verify, k = {k}, half tampered", verify))
    for label, fill in cases:
        for cancel in (False, True):
            secs, dropped, jobs = stop(fill, cancel)
            print(json.dumps({"case": label, "stop": "cancel_all + destroy" if cancel else "destroy (drains)",
                              "seconds_to_destroy_return": round(secs, 4), "dropped": dropped, "jobs": jobs}), flush=True)

    # the abort points' cost: a proof on a pool worker (flag tested, never set) against the bare context (no flag)
    bl = synth.splitmix_blinders(9602)
    want = bytes(PlonkKzgSnark.prove_witness(ctx, pk13, c13.witness, bl)[0])
    pool = ProverPool(0, workers=1)
    try:
        for _ in range(3):  # eager, captured, replayed
            pool.wait(pool.submit_prove_witness(pk13, c13.witness, bl))
        worker, bare = [], []
        for _ in range(args.proofs):
            t0 = time.perf_counter()
            got = pool.wait(pool.submit_prove_witness(pk13, c13.witness, bl))
            worker.append(time.perf_counter() - t0)
            assert bytes(got[0]) == want
            t0 = time.perf_counter()
            PlonkKzgSnark.prove_witness(ctx, pk13, c13.witness, bl)
            bare.append(time.perf_counter() - t0)
    finally:
        pool.close()
    w, b = percentiles(worker), percentiles(bare)
    print(json.dumps({"case": "one 2^13 proof at a time", "pool_worker_flag_tested": w, "bare_context_no_flag": b,
                      "difference_of_medians_ms": round(w["median_ms"] - b["median_ms"], 4)}), flush=True)
    for _, pk in keys.values():
        pk.free()
    bases.free()


if __name__ == "__main__":
    main()
