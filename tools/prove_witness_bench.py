"""Proving from the witness vector (`b200_pool_submit_prove_witness`) against proving from the 5 x n wire table
(`b200_pool_submit_prove`), end to end from host buffers, on one GPU.

    python tools/prove_witness_bench.py [--log-ns 12,14,16] [--ratio 1.4] [--proofs 96] [--repeats 5] [--workers 6]

For each domain size it takes the synthetic circuit of bench.py, pads its witness vector with unused variables to
`--ratio` x n elements (the restated statements have 1.2-1.6 n variables), builds one key from the wiring, and reports:
  * proofs/s through a pool of `--workers` workers with both inputs in pinned host memory: `--repeats` timed windows of
    `--proofs` proofs per path, the two paths alternating, after a warm-up that sizes every worker and captures its
    graphs; median and (min, max) of the windows;
  * the bytes each path copies to the device per proof (computed from the shapes);
  * the gather kernel's device time per proof (torch.profiler, CUDA activities, in a pass of its own);
  * `preprocess_wiring` against `preprocess` on the permutation computed beforehand, median of 3 (host clock around the
    call, which synchronises);
and checks in the same run that both paths give the same proof bytes.  Clocks and power limit are used as found.  One
JSON line per result, headed by the card's name and power limit.
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


def wiring_permutation(wire_vars) -> np.ndarray:
    """The permutation b200_plonk_preprocess_wiring derives: each variable's positions, ascending, form one cycle."""
    v = np.asarray(wire_vars, dtype=np.uint32).reshape(-1)
    order = np.argsort(v, kind="stable")
    sv = v[order]
    nxt = np.roll(order, -1)
    nxt[np.r_[sv[1:] != sv[:-1], True]] = order[np.r_[True, sv[1:] != sv[:-1]]]
    perm = np.empty(v.size, dtype=np.uint64)
    perm[order] = nxt
    return perm


def spread(xs):
    return {"median": statistics.median(xs), "min": min(xs), "max": max(xs)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--log-ns", default="12,14,16")
    ap.add_argument("--ratio", type=float, default=1.4)
    ap.add_argument("--proofs", type=int, default=96)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--workers", type=int, default=6)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("prove_witness_bench: no CUDA device (there is nothing to measure without one)")
    from renegade_b200 import synth
    from renegade_b200.backend import PlonkKzgSnark, ProverPool

    name, power = card()
    print(json.dumps({"card": name, "power_limit,max_sm_clock": power}), flush=True)
    for log_n in (int(x) for x in args.log_ns.split(",")):
        circ = synth.synth_circuit(log_n, num_inputs=8, seed=1)
        n = circ.n
        num_vars = max(circ.num_vars, int(args.ratio * n))
        witness = np.concatenate([circ.witness, synth.splitmix_blinders(log_n, num_vars - circ.num_vars)])
        perm = wiring_permutation(circ.wire_vars)
        row = {"log_n": log_n, "num_vars": num_vars, "num_vars_over_n": num_vars / n,
               "h2d_bytes_per_proof_table": 5 * n * 32 + circ.num_inputs * 32, "h2d_bytes_per_proof_witness": num_vars * 32}

        pool = ProverPool(0, workers=args.workers)
        pc = pool.context(0)
        d_srs = torch.empty((n + 3, 8), dtype=torch.int64, device="cuda")
        pc.known_dlog_bases_device(SEED_SRS, n + 3, d_srs.data_ptr())
        torch.cuda.synchronize()
        bases = pc.load_bases_device(d_srs.data_ptr(), n + 3)

        def timed(fn):
            ts = []
            for _ in range(3):
                t = time.perf_counter()
                fn().free()
                ts.append((time.perf_counter() - t) * 1e3)
            return statistics.median(ts)
        args_pre = (pc, bases, log_n, circ.num_inputs, circ.selectors)
        row["preprocess_ms"] = timed(lambda: PlonkKzgSnark.preprocess(*args_pre, perm, circ.k))
        row["preprocess_wiring_ms"] = timed(lambda: PlonkKzgSnark.preprocess_wiring(*args_pre, circ.wire_vars, num_vars, circ.k))

        pk = PlonkKzgSnark.preprocess_wiring(*args_pre, circ.wire_vars, num_vars, circ.k)
        h_t = torch.from_numpy(np.ascontiguousarray(circ.wires).view(np.int64)).pin_memory()
        h_w = torch.from_numpy(np.ascontiguousarray(witness).view(np.int64)).pin_memory()
        bl = [synth.splitmix_blinders(3000 + i) for i in range(16)]

        def run(path, count):
            if path == "table":
                tks = [pool.submit_prove(pk, h_t.data_ptr(), circ.pub_inputs, bl[i % 16]) for i in range(count)]
                return [bytes(pool.wait(tk)) for tk in tks]
            tks = [pool.submit_prove_witness(pk, h_w.data_ptr(), bl[i % 16]) for i in range(count)]
            return [bytes(pool.wait(tk)[0]) for tk in tks]

        warm = max(4 * args.workers, 16)  # every worker sized, its graphs captured
        row["bytes_equal"] = run("table", warm) == run("witness", warm)
        rates = {"table": [], "witness": []}
        for _ in range(args.repeats):
            for path in ("table", "witness"):
                t = time.perf_counter()
                run(path, args.proofs)
                rates[path].append(args.proofs / (time.perf_counter() - t))
        row["pool_table_proofs_per_s"] = spread(rates["table"])
        row["pool_witness_proofs_per_s"] = spread(rates["witness"])

        # the gather kernel's device time, in a pass of its own (tracing slows the host)
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            run("witness", 16)
            torch.cuda.synchronize()
        hits = [e for e in prof.key_averages() if "k_gather_wires" in e.key]
        row["gather_kernel_us_per_proof"] = (sum(getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0)) for e in hits) /
                                             sum(e.count for e in hits)) if hits else "not measured"
        print(json.dumps(row), flush=True)
        pk.free()
        bases.free()
        pool.close()
        del d_srs
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
