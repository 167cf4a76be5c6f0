"""The express lane (include/b200express.h) under proof load: how long an urgent job takes, submit to result, when it waits
in the FIFO, when it is expedited, and when express workers run it.

    python tools/express_bench.py [--proofs 960] [--repeats 3]

Background load: one pool of 16 normal workers proves the PRIVATE SETTLEMENT (2^12) and OUTPUT BALANCE VALIDITY (2^13)
statements of a private match (examples/host_circuits), alternating, from witness vectors, `--proofs` proofs per window
with 16 in flight.  Foreground: one host thread sends, one after the other, alternating, a private-settlement job with
four hints (`submit_settlement_witness`: the settlement proof and its four link proofs in one job) and a gossip-shaped
verification job (one order: two proofs and their link proof, combined pairing).  Modes:
  fifo      a pool without express workers; foreground jobs are queued behind the load
  expedite  the same pool; every foreground job is expedited right after submit (the front of the line)
  express1  a pool with 1 express worker; every foreground job is expedited onto it
  express2  a pool with 2 express workers; the same
The modes alternate within each of `--repeats` rounds.  Per mode it reports the foreground latency of each job kind,
median / p10 / p90 over every job of every round, and the background proofs/s per window, median (min, max).  Every
foreground result is checked against the bare context's bytes.  Clocks and power limit are used as found; the first
line names the card, its power limit and maximum SM clock.  One JSON line per result.
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
from verify_jobs_bench import seeded_srs  # noqa: E402

MODES = {"fifo": (0, False), "expedite": (0, True), "express1": (1, True), "express2": (2, True)}  # (express, expedite)


def percentiles(xs):
    a = np.asarray(xs, dtype=np.float64)
    return {"median": float(np.median(a)), "p10": float(np.percentile(a, 10)), "p90": float(np.percentile(a, 90)),
            "jobs": int(a.size)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--proofs", type=int, default=960)
    ap.add_argument("--repeats", type=int, default=3)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("express_bench: no CUDA device (there is nothing to measure without one)")
    import renegade_b200 as rb
    from renegade_b200 import synth
    from renegade_b200.backend import PlonkKzgSnark, ProverPool, VerifyingKey, link_proofs

    name, power = card()
    print(json.dumps({"card": name, "power_limit,max_sm_clock": power}), flush=True)
    circs, links = private_match()  # 0 settlement, 1-2 intent and balance validity, 3-4 output balance validity
    ctx = rb.Context(0)  # set-up only: keys made on any context of the device serve every pool's workers
    pts, h, tau_h = seeded_srs(max(c.n for c in circs) + 3)
    bases = ctx.load_bases(pts)
    pks = [PlonkKzgSnark.preprocess_wiring(ctx, bases, c.log_n, c.num_inputs, c.selectors, c.wire_vars, c.num_vars, c.k)
           for c in circs]
    wits = [np.ascontiguousarray(c.witness) for c in circs]
    bl = [synth.splitmix_blinders(9300 + i) for i in range(8)]
    made = [PlonkKzgSnark.prove_witness(ctx, pk, w, bl[j]) for j, (pk, w) in enumerate(zip(pks, wits))]  # (proof, hint, pub)
    settle_links = [(made[a][1], lay) for a, _, lay in links]
    want_settle = PlonkKzgSnark.prove_settlement_witness(ctx, bases, pks[0], wits[0], bl[7], settle_links)
    assert list(want_settle[2]) == [0] * 5
    want_settle = [bytes(want_settle[0])] + [bytes(x) for x in want_settle[1]]
    vks = [VerifyingKey.from_proving_key(pk, h, tau_h) for pk in pks]
    a, b, lay = next(x for x in links if x[0] == 3)
    lp, _ = link_proofs(ctx, bases, made[a][1], made[b][1], lay)
    order = ([vks[a], vks[b]], [made[a][2], made[b][2]], [made[a][0], made[b][0]],
             [(made[a][1].linking_wire_comm, made[b][1].linking_wire_comm, lp, lay)])
    load = [0, 3]  # the background's two statements

    pools = {x: ProverPool(0, workers=16, express=x) for x in (0, 1, 2)}

    def foreground(pool, urgent, kind):
        t0 = time.perf_counter()
        if kind == "settlement":
            t = pool.submit_settlement_witness(bases, pks[0], wits[0], bl[7], settle_links)
        else:
            t = pool.submit_verify(*order, combined=True, g2=(h, tau_h))
        if urgent:
            pool.expedite(t)
        res = pool.wait(t)
        ms = (time.perf_counter() - t0) * 1e3
        if kind == "settlement":
            assert [bytes(res[0])] + [bytes(x) for x in res[1]] == want_settle
        else:
            assert res[0] and all(res[1])
        return ms

    def window(mode, with_foreground=True):
        x, urgent = MODES[mode]
        pool = pools[x]
        done, lat = threading.Event(), {"settlement": [], "verify": []}

        def stream():
            i = 0
            while not done.is_set():
                kind = ("settlement", "verify")[i % 2]
                lat[kind].append(foreground(pool, urgent, kind))
                i += 1

        th = threading.Thread(target=stream) if with_foreground else None
        t0 = time.perf_counter()
        if th:
            th.start()
        inflight, i = [], 0
        while i < args.proofs or inflight:
            while i < args.proofs and len(inflight) < 16:
                j = load[i % 2]
                inflight.append(pool.submit_prove_witness(pks[j], wits[j], bl[i % 8]))
                i += 1
            pool.wait(inflight.pop(0))
        rate = args.proofs / (time.perf_counter() - t0)
        done.set()
        if th:
            th.join()
        return rate, lat

    # warm-up: every worker, express ones included, has proved both load keys and run both foreground kinds
    for mode in MODES:
        window(mode)
    for x, pool in pools.items():
        for _ in range(4 * (x + 1)):
            for kind in ("settlement", "verify"):
                foreground(pool, True, kind)
    rates, lats = {}, {}
    for _ in range(args.repeats):
        for mode in MODES:
            r, lat = window(mode)
            rates.setdefault(mode, []).append(r)
            for kind, xs in lat.items():
                lats.setdefault((mode, kind), []).extend(xs)
    for mode in MODES:
        print(json.dumps({"mode": mode, "express_workers": MODES[mode][0], "expedite": MODES[mode][1],
                          "settlement_ms": percentiles(lats[(mode, "settlement")]),
                          "verify_ms": percentiles(lats[(mode, "verify")]),
                          "background_proofs_per_s": spread(rates[mode])}), flush=True)
    for pool in pools.values():
        pool.close()
    for pk in pks:
        pk.free()
    bases.free()
    ctx.close()


if __name__ == "__main__":
    main()
