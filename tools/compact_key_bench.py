"""Default versus compact proving keys (include/b200compact.h): one proof at a time, eager and from replayed graphs, and
proofs/s through a pool, with preprocessing's device bytes and the context's peak.

    python tools/compact_key_bench.py [--sizes 16,20,22,23] [--reps 10] [--pool-proofs 120] [--out FILE]

Each size and mode runs on a context of its own: an SRS of n + 3 known-discrete-log points made on the device (timing
only: these proofs are not meant to verify), the satisfied circuit of tests/large_domains.py, one key, then `reps`
proofs with graphs off (eager) and `reps` with graphs on after two warm-up proofs (replayed).  The compact key's
replayed proof must have the default key's bytes.  Preprocessing bytes and peak context bytes are free device memory
before minus after (meaningful on an otherwise idle GPU): preprocessing's growth (the key and the scratch it reserves) and the
context's peak, next to b200_plonk_footprint's estimates of the key and of the whole context.  The pool leg runs 2^16
witness-vector proofs through a pool of 6 workers.  Prints one JSON line per measurement (and writes them to --out)."""
import argparse
import gc
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
import large_domains as ld  # noqa: E402
import renegade_b200 as rb  # noqa: E402
from renegade_b200 import synth  # noqa: E402
from renegade_b200.backend import PlonkKzgSnark, ProverPool  # noqa: E402


def free_bytes():
    gc.collect()
    torch.cuda.empty_cache()
    return torch.cuda.mem_get_info()[0]


def stats(ts):
    a = np.array(ts) * 1e3
    return {"median_ms": float(np.median(a)), "p10_ms": float(np.percentile(a, 10)), "p90_ms": float(np.percentile(a, 90)),
            "n": len(ts)}


def device_srs(ctx, n, seed=0xB200):
    buf = torch.empty(n * 64, dtype=torch.uint8, device="cuda")
    ctx.known_dlog_bases_device(seed, n, buf.data_ptr())
    torch.cuda.synchronize()
    bases = ctx.load_bases_device(buf.data_ptr(), n)
    del buf
    return bases


def one_size(circ, log_n, compact, reps):
    free0 = free_bytes()
    low = [free0]

    def note():
        low.append(torch.cuda.mem_get_info()[0])

    ctx = rb.Context(0)
    try:
        bases = device_srs(ctx, (1 << log_n) + 3)
        f1 = free_bytes()
        t0 = time.perf_counter()
        pk = PlonkKzgSnark.preprocess(ctx, bases, log_n, circ.num_inputs, circ.selectors, circ.perm, circ.k, compact=compact)
        t_key = time.perf_counter() - t0
        preprocess_bytes = f1 - free_bytes()  # the key and the NTT and MSM scratch preprocessing grows
        bl = synth.splitmix_blinders(0xBE4C)
        out = {}
        for name, graphs, warm in (("eager", False, 1), ("replayed", True, 2)):
            ctx.use_graphs(graphs)
            for _ in range(warm):
                PlonkKzgSnark.prove_with_link_hint(ctx, pk, circ.wires, circ.pub_inputs, bl)
                note()
            ts = []
            for _ in range(reps):
                t0 = time.perf_counter()
                proof = PlonkKzgSnark.prove_with_link_hint(ctx, pk, circ.wires, circ.pub_inputs, bl)[0]
                ts.append(time.perf_counter() - t0)
                note()
            out[name] = stats(ts)
        est = PlonkKzgSnark.footprint(log_n, 1, compact)
        res = {"log_n": log_n, "mode": "compact" if compact else "default", **{f"{k}_{s}": v for k, d in out.items()
                                                                              for s, v in d.items()},
               "preprocess_s": t_key, "preprocess_bytes": preprocess_bytes, "key_bytes_estimate": est["key"],
               "peak_context_bytes": free0 - min(low), "estimate_bytes": sum(est.values())}
        digest = bytes(proof)
        pk.free()
        bases.free()
    finally:
        ctx.close()
    return res, digest


def pool_leg(compact, proofs, workers=6):
    log_n = 16
    circ = ld.big_circuit(log_n, seed=0x16)
    pool = ProverPool(0, workers=workers)
    try:
        ctx = pool.context(0)
        bases = device_srs(ctx, (1 << log_n) + 3)
        wpk = PlonkKzgSnark.preprocess_wiring(ctx, bases, log_n, circ.num_inputs, circ.selectors, circ.wire_vars, circ.num_vars,
                                              circ.k, compact=compact)
        bls = [synth.splitmix_blinders(0x9000 + i) for i in range(proofs)]
        for t in [pool.submit_prove_witness(wpk, circ.witness, bls[i]) for i in range(2 * workers)]:
            pool.wait(t)
        t0 = time.perf_counter()
        tickets = [pool.submit_prove_witness(wpk, circ.witness, b) for b in bls]
        for t in tickets:
            pool.wait(t)
        dt = time.perf_counter() - t0
        wpk.free()
        bases.free()
    finally:
        pool.close()
    return {"leg": "pool", "log_n": log_n, "mode": "compact" if compact else "default", "workers": workers, "proofs": proofs,
            "proofs_per_s": proofs / dt}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="16,20,22,23")
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--pool-proofs", type=int, default=120)
    ap.add_argument("--out", default=None, help="also write the JSON lines to this file")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("compact_key_bench: no CUDA device")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()[0]
    rows = [{"gpu": gpu}]
    print(json.dumps(rows[0]), flush=True)
    for log_n in (int(s) for s in a.sizes.split(",")):
        t0 = time.time()
        circ = ld.big_circuit(log_n, seed=log_n)
        print(f"# 2^{log_n}: circuit in {time.time() - t0:.1f} s", flush=True)
        digests = {}
        for compact in ((False, True) if log_n <= 22 else (True,)):
            need = sum(PlonkKzgSnark.footprint(log_n, 1, compact).values())
            if free_bytes() < need:
                row = {"log_n": log_n, "mode": "compact" if compact else "default", "skipped": "free memory below the estimate",
                       "estimate_bytes": need}
            else:
                row, digests[compact] = one_size(circ, log_n, compact, a.reps)
            rows.append(row)
            print(json.dumps(row), flush=True)
        if len(digests) == 2:
            assert digests[True] == digests[False], f"2^{log_n}: compact and default proofs differ"
    for compact in (False, True, False, True):  # alternated
        row = pool_leg(compact, a.pool_proofs)
        rows.append(row)
        print(json.dumps(row), flush=True)
    if a.out:
        with open(a.out, "w") as f:
            f.write("".join(json.dumps(r) + "\n" for r in rows))


if __name__ == "__main__":
    main()
