"""Time b200_srs_check on 2^17 + 3 seeded powers (the prover's full SRS size, MAX_SRS_DEGREE + 1) in its two parts:

  * the combined check of a valid SRS: weights, one batch-2 MSM over the resident bases, the host pairing, plus the
    generator read-back and the two G2 subgroup tests on the host (the MSM's device time and the subgroup tests are
    also timed on their own);
  * the locate pass: every consecutive pair checked on its own on the device, timed as a failing check with locate
    minus the same check without it.

    python tools/srs_check_bench.py [--log-n 17] [--reps 10] [--out FILE.json]

Each figure is the median of `reps` calls after one warm-up call of the same shape; every call ends in a device
synchronise.  The powers come from the C oracle (a fixed tau), so the numbers can be re-run exactly.  Needs a CUDA
device."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))

import bn254_pairing_py as pr  # noqa: E402
import bn254_py as py  # noqa: E402
import oracle_c  # noqa: E402
import renegade_b200 as rb  # noqa: E402
from renegade_b200.backend import g2_in_subgroup  # noqa: E402

TAU = 0x1D2C3B4A59687706F5E4D3C2B1A09F8E7D6C5B4A39281706F5E4D3C2B1A0987


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def median_ms(fn, reps):
    fn()  # warm-up: the MSM scratch and the module's kernels
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        ts.append((time.perf_counter() - t0) * 1e3)
    return statistics.median(ts), min(ts), max(ts)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--log-n", type=int, default=17)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default=None, help="also write the results here (JSON)")
    args = ap.parse_args()
    n = (1 << args.log_n) + 3
    oracle_c.build()
    pts = oracle_c.srs_from_tau(oracle_c.int_to_limbs(py.to_mont(TAU % py.R, py.R)), n)
    raw = np.frombuffer(open(os.path.join(ROOT, "tests", "golden", "srs_g2.bin"), "rb").read(), dtype=np.uint64)
    h = raw[:16].copy()
    tau_h = np.frombuffer(pr.encode_g2_mont(pr.g2_mul(pr.decode_g2_mont(h.tobytes(), 0), TAU % pr.R)), dtype=np.uint64).copy()
    ctx = rb.Context(0)
    bases = ctx.load_bases(pts)
    seed = bytes(range(32))
    rep = rb.check_srs(ctx, bases, h, tau_h, seed=seed)
    assert rep.valid, rep
    bad = rb.check_srs(ctx, bases, tau_h, h, seed=seed)  # swapped pair: every pair fails
    assert bad.n_bad == n - 1, bad
    combined = median_ms(lambda: rb.check_srs(ctx, bases, h, tau_h, seed=seed), args.reps)
    subgroup = median_ms(lambda: (g2_in_subgroup(h), g2_in_subgroup(tau_h)), args.reps)
    failed = median_ms(lambda: rb.check_srs(ctx, bases, tau_h, h, seed=seed, locate=False), args.reps)
    located = median_ms(lambda: rb.check_srs(ctx, bases, tau_h, h, seed=seed, locate=True), max(3, args.reps // 3))
    locate_ms = located[0] - failed[0]
    ctx.msm_timing(True)  # device time of the check's batch-2 MSM (CUDA events on the context's stream)
    msm_ms = []
    for _ in range(args.reps):
        rb.check_srs(ctx, bases, h, tau_h, seed=seed)
        msm_ms.append(ctx.msm_timing(True)["total"])
    ctx.msm_timing(False)
    res = {
        "card": card(),
        "n_powers": n,
        "combined_check_ms": {"median": combined[0], "min": combined[1], "max": combined[2]},
        "msm_device_ms_median": statistics.median(msm_ms),
        "g2_subgroup_tests_ms": {"median": subgroup[0], "min": subgroup[1], "max": subgroup[2]},
        "failed_check_without_locate_ms": {"median": failed[0], "min": failed[1], "max": failed[2]},
        "failed_check_with_locate_ms": {"median": located[0], "min": located[1], "max": located[2]},
        "locate_pass_ms": locate_ms,
        "locate_pairs_per_s": (n - 1) / (locate_ms / 1e3),
    }
    print(json.dumps(res, indent=1))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)
    bases.free()
    ctx.close()


if __name__ == "__main__":
    main()
