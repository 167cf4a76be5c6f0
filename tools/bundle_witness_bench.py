"""Private-match bundles from witness vectors (`b200_pool_submit_bundle_witness`) against bundles from 5 x n wire tables
(`b200_pool_submit_bundle`), end to end through one pool on one GPU.

    python tools/bundle_witness_bench.py [--bundles 24] [--repeats 5] [--workers 6]

The bundle is the private match of bench.py's private_match_bundle leg: the restated PRIVATE SETTLEMENT (2^12), two
INTENT AND BALANCE VALIDITY (2^14) and two OUTPUT BALANCE VALIDITY (2^13) statements of examples/host_circuits with the
four link proofs, every key made from the circuit's wiring (so both paths prove under the same key).  It reports:
  * bundles/s for each path with its inputs in pinned host memory: `--repeats` timed windows of `--bundles` bundles
    per path, the two paths alternating, after a warm-up that sizes every worker and captures its graphs; median and
    (min, max) of the windows;
  * the bytes each path copies to the device per bundle (from the shapes);
  * the host time to build one bundle's inputs: the five 5 x n tables gathered from the witness vectors against the five
    witness vectors copied as they are, both into pinned buffers (median of 20);
and checks in the same run that both paths give the same proof and link-proof bytes.  Clocks and power limit are used
as found.  One JSON line per result, headed by the card's name and power limit.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "examples"))

import numpy as np  # noqa: E402

SEED_SRS = 0x5EED


def card():
    try:
        import torch
        name = torch.cuda.get_device_name(0)
    except Exception:
        name = "unknown"
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        out = "unknown"
    return name, out


def private_match():
    """The five circuits and four links (validity proof j <-> settlement proof 0) of bench.py's private_match_bundle leg."""
    from host_circuits import intent_and_balance_validity as val
    from host_circuits import output_balance_validity as obv
    from host_circuits import private_settlement as ps
    from renegade_b200.backend import GroupLayout
    parties, _ = ps.create_witness_statement(seed=61)
    validity = [val.create_witness_statement(seed=70 + i, intent=parties[i].intent, balance=parties[i].input_balance)
                for i in (0, 1)]
    out_validity = [obv.create_witness_statement(80 + i, parties[i].output_balance) for i in (0, 1)]
    parties, statement = ps.create_witness_statement(
        seed=61, linked=[(validity[i][0].new_amount_public_share, validity[i][0].post_match_balance_shares,
                          out_validity[i][0].post_match_balance_shares) for i in (0, 1)])
    settlement_cs = ps.IntentAndBalancePrivateSettlementCircuit.build(parties, statement)
    layouts = settlement_cs.get_circuit_layout()
    circs = [settlement_cs.finalize_for_arithmetization()] + \
            [val.IntentAndBalanceValidityCircuit.build(w, st, layouts).finalize_for_arithmetization() for w, st in validity] + \
            [obv.OutputBalanceValidityCircuit.build(w, st, layouts).finalize_for_arithmetization() for w, st in out_validity]
    lay = lambda g: GroupLayout(layouts[g].alignment, layouts[g].offset, layouts[g].size)  # noqa: E731
    links = [(1 + p, 0, lay(g)) for p, g in enumerate(ps.PARTY_LINKS)] + \
            [(3 + p, 0, lay(g)) for p, g in enumerate(ps.OUTPUT_LINKS)]
    return circs, links


def spread(xs):
    return {"median": statistics.median(xs), "min": min(xs), "max": max(xs)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--bundles", type=int, default=24)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--workers", type=int, default=6)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("bundle_witness_bench: no CUDA device (there is nothing to measure without one)")
    from renegade_b200 import synth
    from renegade_b200.backend import PlonkKzgSnark, ProverPool

    name, power = card()
    print(json.dumps({"card": name, "power_limit,max_sm_clock": power}), flush=True)
    circs, links = private_match()
    n_max = max(c.n for c in circs)
    row = {"statements": [{"log_n": c.log_n, "num_vars": c.num_vars, "num_inputs": c.num_inputs} for c in circs],
           "links": len(links),
           "h2d_bytes_per_bundle_table": sum(5 * c.n * 32 + c.num_inputs * 32 for c in circs),
           "h2d_bytes_per_bundle_witness": sum(c.num_vars * 32 for c in circs)}

    # host work per bundle: the five tables gathered from the witness vectors, against the witness vectors as they are
    pin = lambda shape: torch.empty(shape, dtype=torch.int64).pin_memory().numpy().view(np.uint64)  # noqa: E731
    h_t = [pin((5, c.n, 4)) for c in circs]
    h_w = [pin((c.num_vars, 4)) for c in circs]

    def build_tables():
        for c, t in zip(circs, h_t):
            np.take(c.witness, c.wire_vars, axis=0, out=t)

    def build_witnesses():
        for c, w in zip(circs, h_w):
            np.copyto(w, c.witness)

    for what, fn in (("host_build_ms_per_bundle_table", build_tables), ("host_build_ms_per_bundle_witness", build_witnesses)):
        ts = []
        for _ in range(20):
            t = time.perf_counter()
            fn()
            ts.append((time.perf_counter() - t) * 1e3)
        row[what] = statistics.median(ts)
    assert all((t == c.wires).all() for t, c in zip(h_t, circs))

    pool = ProverPool(0, workers=args.workers)
    pc = pool.context(0)
    d_srs = torch.empty((n_max + 3, 8), dtype=torch.int64, device="cuda")
    pc.known_dlog_bases_device(SEED_SRS, n_max + 3, d_srs.data_ptr())
    torch.cuda.synchronize()
    bases = pc.load_bases_device(d_srs.data_ptr(), n_max + 3)
    pks = [PlonkKzgSnark.preprocess_wiring(pc, bases, c.log_n, c.num_inputs, c.selectors, c.wire_vars, c.num_vars, c.k)
           for c in circs]
    bl = [synth.splitmix_blinders(7000 + i) for i in range(8)]

    def run(path, count):
        if path == "table":
            tks = [pool.submit_bundle(bases, [(pks[j], h_t[j].ctypes.data, circs[j].pub_inputs, bl[(5 * b + j) % 8])
                                              for j in range(5)], links) for b in range(count)]
        else:
            tks = [pool.submit_bundle_witness(bases, [(pks[j], h_w[j].ctypes.data, bl[(5 * b + j) % 8]) for j in range(5)],
                                              links) for b in range(count)]
        return [[bytes(p) for p in r[0]] + [bytes(lp) for lp in r[2]] for r in (pool.wait(tk) for tk in tks)]

    warm = max(2, args.workers)  # every worker has proved every key more than once (buffers sized, graphs captured)
    row["bytes_equal"] = run("table", warm) == run("witness", warm)
    rates = {"table": [], "witness": []}
    for _ in range(args.repeats):
        for path in ("table", "witness"):
            t = time.perf_counter()
            run(path, args.bundles)
            rates[path].append(args.bundles / (time.perf_counter() - t))
    row["pool_table_bundles_per_s"] = spread(rates["table"])
    row["pool_witness_bundles_per_s"] = spread(rates["witness"])
    row["workers"] = args.workers
    print(json.dumps(row), flush=True)
    for pk in pks:
        pk.free()
    bases.free()
    pool.close()


if __name__ == "__main__":
    main()
