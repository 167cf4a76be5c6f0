"""Reserved SMs for the express lane (include/b200reserved.h) under proof load: how long an urgent job takes, submit to
result, and what the load loses, when the express worker runs on SMs of its own.

    python tools/reserved_bench.py [--proofs 1920] [--repeats 3]

Load and foreground as in tools/express_bench.py: a pool of 16 normal workers proves the PRIVATE SETTLEMENT (2^12) and
OUTPUT BALANCE VALIDITY (2^13) statements of a private match from witness vectors, alternating, `--proofs` proofs per
window with 16 in flight; one host thread sends, one after the other, alternating, a private-settlement job with four
hints and a gossip-shaped verification job (combined pairing).  Modes:
  fifo        a pool without express workers; foreground jobs are queued behind the load
  expedite    the same pool; every foreground job is expedited right after submit (the front of the line)
  express     a pool with 1 express worker on the same SMs as the load (stream priorities only); jobs expedited onto it
  reserved8   a pool with 1 express worker on a reserved group of at least 8 SMs, the load on the rest; the same
  reserved16  the same with 16 SMs
  reserved24  the same with 24 SMs
The modes alternate within each of `--repeats` rounds.  Per mode it reports the foreground latency of each job kind,
median / p10 / p90 over every job of every round, the background proofs/s per window, median (min, max), and the
partition as the split rounded it.  Every foreground result is checked against the bare context's bytes in the same
run.  Clocks and power limit are used as found; the first line names the card, its power limit and maximum SM clock.
One JSON line per result.
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
from express_bench import percentiles  # noqa: E402
from verify_jobs_bench import seeded_srs  # noqa: E402

# (express workers, expedite, reserved SMs)
MODES = {"fifo": (0, False, 0), "expedite": (0, True, 0), "express": (1, True, 0), "reserved8": (1, True, 8),
         "reserved16": (1, True, 16), "reserved24": (1, True, 24)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--proofs", type=int, default=1920)
    ap.add_argument("--repeats", type=int, default=3)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("reserved_bench: no CUDA device (there is nothing to measure without one)")
    import renegade_b200 as rb
    from renegade_b200 import synth
    from renegade_b200.backend import PlonkKzgSnark, ProverPool, VerifyingKey, link_proofs

    name, power = card()
    print(json.dumps({"card": name, "power_limit,max_sm_clock": power,
                      "sms": torch.cuda.get_device_properties(0).multi_processor_count}), flush=True)
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
    want_verdict = PlonkKzgSnark.batch_verify(ctx, *order, g2=(h, tau_h))
    load = [0, 3]  # the background's two statements

    pools = {}
    for mode, (x, _, sms) in MODES.items():
        if mode != "expedite":  # fifo and expedite share one pool
            pools[mode] = ProverPool(0, workers=16, express=x, express_sms=sms)
    pools["expedite"] = pools["fifo"]
    checked = {"settlement": 0, "verify": 0}

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
            assert res[0] and all(res[1]) and (res[0], list(res[1])) == (want_verdict[0], list(want_verdict[1]))
        checked[kind] += 1
        return ms

    def window(mode):
        pool, urgent = pools[mode], MODES[mode][1]
        done, lat = threading.Event(), {"settlement": [], "verify": []}

        def stream():
            i = 0
            while not done.is_set():
                kind = ("settlement", "verify")[i % 2]
                lat[kind].append(foreground(pool, urgent, kind))
                i += 1

        th = threading.Thread(target=stream)
        t0 = time.perf_counter()
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
        th.join()
        return rate, lat

    # warm-up: every worker, express ones included, has proved both load keys and run both foreground kinds
    for mode in MODES:
        window(mode)
    for mode in MODES:
        for _ in range(4):
            for kind in ("settlement", "verify"):
                foreground(pools[mode], True, kind)
    rates, lats = {}, {}
    for _ in range(args.repeats):
        for mode in MODES:
            r, lat = window(mode)
            rates.setdefault(mode, []).append(r)
            for kind, xs in lat.items():
                lats.setdefault((mode, kind), []).extend(xs)
    for mode, (x, urgent, sms) in MODES.items():
        normal, express = pools[mode].partition()
        print(json.dumps({"mode": mode, "express_workers": x, "expedite": urgent, "express_sms": sms,
                          "partition_normal_express": [normal, express],
                          "settlement_ms": percentiles(lats[(mode, "settlement")]),
                          "verify_ms": percentiles(lats[(mode, "verify")]),
                          "background_proofs_per_s": spread(rates[mode])}), flush=True)
    print(json.dumps({"bytes_equal": True, "foreground_jobs_checked": checked}), flush=True)
    for mode, pool in pools.items():
        if mode != "expedite":
            pool.close()
    for pk in pks:
        pk.free()
    bases.free()
    ctx.close()


if __name__ == "__main__":
    main()
