"""Settlement jobs (`b200_pool_submit_settlement[_witness]`) against the two-step path a caller without them takes: prove,
wait on the host, then submit the link proofs.

    python tools/settlement_bench.py [--lone 15] [--per-thread 8] [--repeats 3]

Shapes (examples/host_circuits): the PRIVATE SETTLEMENT (2^12) against four validity hints (2^14 + 2 and 2^13 + 2), and
the INTENT ONLY PUBLIC SETTLEMENT (2^9) against one INTENT ONLY VALIDITY hint (2^13 + 2).  The hints are made once, before
anything is timed, as a relayer keeps them from the validity proofs made when the order was placed.  Paths:
  A    submit_prove + wait + submit_link_batch + wait
  A'   submit_prove + wait + k x submit_link + wait (the service's path without settlement jobs)
  B    submit_settlement
  B-w  submit_settlement_witness
Every key is made from the circuit's wiring, so all paths prove under one key; inputs sit in pinned host memory.
It reports, per shape and path:
  * the latency of one settlement alone on an idle pool of 6 workers: `--lone` runs per path, the paths alternating,
    median (min, max) in ms;
  * settlements/s with 16 in flight on a pool of 16 workers: 16 host threads, each making `--per-thread` settlements one
    after the other, `--repeats` windows per path, the paths alternating; median (min, max);
and checks in the same run that every path returns the same proof and link-proof bytes.  Clocks and power limit are
used as found.  One JSON line per result, headed by the card's name and power limit.
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
sys.path.insert(0, os.path.join(ROOT, "tools"))

import numpy as np  # noqa: E402

from bundle_witness_bench import card, private_match, spread  # noqa: E402

SEED_SRS = 0x5EED
PATHS = ("A", "A'", "B", "B-w")


def intent_only():
    from host_circuits import intent_only as io
    from renegade_b200.backend import GroupLayout
    intent = io.create_public_settlement_witness_statement(51)[0].intent
    settlement = io.IntentOnlyPublicSettlementCircuit.build(*io.create_public_settlement_witness_statement(54, intent))
    lay = settlement.get_circuit_layout()[io.INTENT_ONLY_SETTLEMENT_LINK]
    validity = io.IntentOnlyValidityCircuit.build(*io.create_validity_witness_statement(52, intent), lay)
    return [settlement.finalize_for_arithmetization(), validity.finalize_for_arithmetization()], \
        [(1, 0, GroupLayout(lay.alignment, lay.offset, lay.size))]


class Shape:
    """One settlement shape on one pool: keys, pinned inputs, the stored hints."""

    def __init__(self, name, circs, links, pool, torch):
        from renegade_b200 import synth
        from renegade_b200.backend import PlonkKzgSnark
        self.name, self.circs, self.pool = name, circs, pool
        pc = pool.context(0)
        n_max = max(c.n for c in circs)
        d_srs = torch.empty((n_max + 3, 8), dtype=torch.int64, device="cuda")
        pc.known_dlog_bases_device(SEED_SRS, n_max + 3, d_srs.data_ptr())
        torch.cuda.synchronize()
        self.bases = pc.load_bases_device(d_srs.data_ptr(), n_max + 3)
        self.pks = [PlonkKzgSnark.preprocess_wiring(pc, self.bases, c.log_n, c.num_inputs, c.selectors, c.wire_vars,
                                                    c.num_vars, c.k) for c in circs]
        pin = lambda a: (lambda t: (np.copyto(t, a), t)[1])(  # noqa: E731
            torch.empty(a.shape, dtype=torch.int64).pin_memory().numpy().view(np.uint64))
        c0 = circs[0]
        self.table, self.witness = pin(np.ascontiguousarray(c0.wires)), pin(np.ascontiguousarray(c0.witness))
        self.bl = [synth.splitmix_blinders(7000 + i) for i in range(8)]
        self.links = []
        for a, _, lay in links:
            _, hint, _ = PlonkKzgSnark.prove_witness(pc, self.pks[a], circs[a].witness, self.bl[a])
            self.links.append((hint, lay))

    def run(self, path, i):
        """One settlement by `path` with blinder set i: bytes of the proof and the link proofs."""
        p, pk, c0, bl = self.pool, self.pks[0], self.circs[0], self.bl[i % 8]
        if path == "B":
            proof, lps, st = p.wait(p.submit_settlement(self.bases, pk, self.table.ctypes.data, c0.pub_inputs, bl, self.links))
        elif path == "B-w":
            proof, lps, st, _ = p.wait(p.submit_settlement_witness(self.bases, pk, self.witness.ctypes.data, bl, self.links))
        else:
            from renegade_b200.backend import LinkingHint
            proof, poly = p.wait(p.submit_prove(pk, self.table.ctypes.data, c0.pub_inputs, bl, with_link_poly=True))
            hint = LinkingHint(poly, np.array(proof.wires_poly_comms[0], dtype=np.uint64))
            if path == "A":
                lps, _, st = p.wait(p.submit_link_batch(self.bases, [(h, hint, lay) for h, lay in self.links]))
                st = [0] + st
            else:
                lps = [p.wait(t) for t in [p.submit_link(self.bases, h, hint, lay) for h, lay in self.links]]
                st = [0] * (len(lps) + 1)
        assert not any(st), (path, st)
        return [bytes(proof)] + [bytes(x) for x in lps]

    def free(self):
        for pk in self.pks:
            pk.free()
        self.bases.free()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lone", type=int, default=15)
    ap.add_argument("--per-thread", type=int, default=8)
    ap.add_argument("--repeats", type=int, default=3)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("settlement_bench: no CUDA device (there is nothing to measure without one)")
    from renegade_b200.backend import ProverPool

    name, power = card()
    print(json.dumps({"card": name, "power_limit,max_sm_clock": power}), flush=True)
    shapes = (("private", private_match()), ("intent_only", intent_only()))
    for workers, mode in ((6, "lone"), (16, "throughput")):
        pool = ProverPool(0, workers=workers)
        for sname, (circs, links) in shapes:
            s = Shape(sname, circs, links, pool, torch)
            row = {"shape": sname, "mode": mode, "workers": workers, "links": len(s.links),
                   "log_n": [c.log_n for c in circs]}
            # warm-up: every worker has run every path more than once (buffers sized, graphs captured); bytes checked
            outs = {path: [s.run(path, i) for i in range(2 * workers)] for path in PATHS}
            row["bytes_equal"] = all(outs[path] == outs["A'"] for path in PATHS)
            if mode == "lone":
                ms = {path: [] for path in PATHS}
                for i in range(args.lone):
                    for path in PATHS:
                        t = time.perf_counter()
                        s.run(path, i)
                        ms[path].append((time.perf_counter() - t) * 1e3)
                row["lone_ms"] = {path: spread(v) for path, v in ms.items()}
            else:
                rates = {path: [] for path in PATHS}
                for _ in range(args.repeats):
                    for path in PATHS:
                        def worker(t0):
                            for i in range(args.per_thread):
                                s.run(path, t0 + i)
                        threads = [threading.Thread(target=worker, args=(k,)) for k in range(16)]
                        t = time.perf_counter()
                        for th in threads:
                            th.start()
                        for th in threads:
                            th.join()
                        rates[path].append(16 * args.per_thread / (time.perf_counter() - t))
                row["settlements_per_s"] = {path: spread(v) for path, v in rates.items()}
            print(json.dumps(row), flush=True)
            s.free()
        pool.close()


if __name__ == "__main__":
    main()
