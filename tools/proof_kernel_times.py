"""Per-kernel GPU time of the benchmark's proof (n = 2^16 synthetic circuit, `synth.synth_circuit(16, 17, 0xB200)`).

Proves K proofs under torch.profiler (CUDA activities) in two modes, one proof at a time on one context and
`--workers` in flight through `ProverPool`, and prints per kernel: launches per proof, GPU time per proof and share of
the kernel time.  With proofs in flight the kernels overlap, so a kernel's time there is its own duration on a shared
GPU, not wall time.  A third pass proves K more through the pool with the profiler off and reports proofs/s.  The card's
name, power limit and max SM clock are printed with the tables.

    python tools/proof_kernel_times.py [--proofs 50] [--workers 6] [--window-bits 0] [--json OUT]

`--window-bits` is the MSM window of the SRS bases (0: the throughput plan the prover uses, >= 2: that window c).
"""
import argparse
import collections
import json
import os
import subprocess
import sys
import tempfile
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
from torch.profiler import ProfilerActivity, profile

import renegade_b200 as rb
from renegade_b200 import synth
from renegade_b200.backend import PlonkKzgSnark, ProverPool, prove_raw

LOG_N, NUM_INPUTS, CIRCUIT_SEED = 16, 17, 0xB200


def card_info() -> dict:
    info = {"name": torch.cuda.get_device_name(0)}
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout.strip().split(", ")
        info.update(name=out[0], power_limit_w=float(out[1]), sm_max_mhz=float(out[2]))
    except (OSError, IndexError, ValueError, subprocess.SubprocessError):
        info.update(power_limit_w=None, sm_max_mhz=None)
    return info


def short(name: str) -> str:
    for junk in ("void ", "b200::", "(anonymous namespace)::", "<unnamed>::"):
        name = name.replace(junk, "")
    return name.split("(")[0].split("<")[0].strip()


def kernel_table(run, proofs: int) -> dict:
    """Runs `run()` under the profiler; returns {kernel: (launches per proof, us per proof)} from the trace's kernel events."""
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        run()
        torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "trace.json")
        prof.export_chrome_trace(path)
        events = json.load(open(path))["traceEvents"]
    agg = collections.defaultdict(lambda: [0, 0.0])
    for e in events:
        if e.get("cat") == "kernel" and e.get("ph") == "X":
            a = agg[short(e["name"])]
            a[0] += 1
            a[1] += float(e["dur"])
    if not agg:
        sys.exit("the profiler recorded no kernels")
    return {k: (c / proofs, us / proofs) for k, (c, us) in agg.items()}


def print_table(title: str, table: dict) -> None:
    total = sum(us for _, us in table.values())
    launches = sum(c for c, _ in table.values())
    print(f"\n## {title}: {launches:.1f} launches, {total:.1f} us of kernel time per proof")
    print(f"{'kernel':44s} {'launches':>9s} {'us/proof':>10s} {'share':>7s}")
    for k, (c, us) in sorted(table.items(), key=lambda kv: -kv[1][1]):
        print(f"{k:44s} {c:9.2f} {us:10.1f} {100 * us / total:6.1f}%")


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--proofs", type=int, default=50)
    ap.add_argument("--workers", type=int, default=6)
    ap.add_argument("--window-bits", type=int, default=0)
    ap.add_argument("--json", help="also write the tables and the card as JSON to this path")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("needs a CUDA device")
    K, conc = args.proofs, args.workers
    n = 1 << LOG_N
    pool = ProverPool(0, workers=conc)
    ctx = pool.context(0)
    circ = synth.synth_circuit(LOG_N, num_inputs=NUM_INPUTS, seed=CIRCUIT_SEED)
    d_srs = torch.empty((n + 3, 8), dtype=torch.int64, device="cuda")
    torch.cuda.synchronize()
    ctx.known_dlog_bases_device(0x7A0, n + 3, d_srs.data_ptr())  # any valid G1 points cost what the real SRS costs
    srs = ctx.load_bases_device(d_srs.data_ptr(), n + 3, window_bits=args.window_bits)
    pk = PlonkKzgSnark.preprocess(ctx, srs, LOG_N, circ.num_inputs, circ.selectors, circ.perm, circ.k)
    d_wires = torch.from_numpy(circ.wires.view(np.int64)).cuda()
    torch.cuda.synchronize()
    blinders = [synth.splitmix_blinders(i) for i in range(8)]

    def serial(count):
        for i in range(count):
            prove_raw(ctx, pk, d_wires.data_ptr(), circ.pub_inputs, blinders[i % 8])

    def pooled(count):
        tickets = [pool.submit_prove(pk, d_wires.data_ptr(), circ.pub_inputs, blinders[i % 8]) for i in range(count)]
        for tk in tickets:
            pool.wait(tk)

    # warm-up: every worker captures its rounds as graphs and replays them before anything is profiled
    serial(3)
    for _ in range(3):
        pooled(conc)
    tables = {"one proof at a time": kernel_table(lambda: serial(K), K),
              f"{conc} in flight through ProverPool": kernel_table(lambda: pooled(K), K)}
    pooled(conc)
    t = time.perf_counter()
    pooled(K)
    rate = K / (time.perf_counter() - t)
    card = card_info()
    print(f"# {card['name']}, power limit {card['power_limit_w']} W, max SM clock {card['sm_max_mhz']} MHz; "
          f"n = 2^{LOG_N}, MSM plan {srs.plan}, {K} proofs per table")
    for title, table in tables.items():
        print_table(title, table)
    print(f"\n{conc} in flight, profiler off: {rate:.1f} proofs/s")
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"card": card, "plan": srs.plan, "proofs": K, "proofs_per_s": rate,
                       "tables": {t: {k: {"launches": c, "us": us} for k, (c, us) in tab.items()} for t, tab in tables.items()}}, f, indent=1)
    pool.close()


if __name__ == "__main__":
    main()
