"""Latency of the device pairing checks for a few items against many: b200_pairing_check_many (m = 2) over n checks and
b200_plonk_verify_each over k proofs (2^7 gates, 4 public inputs, the reference's SRS head, the proofs
tools/verify_each_bench.py builds), with none and with a quarter of them tampered; and the kernels of one small call by
torch.profiler (k_pairing_warp / k_pairing_many, k_prepare, k_item_points).

    python tools/verify_latency_bench.py [--parent DIR] [--rounds 3] [--reps 5] [--out FILE.json]

With --parent (a built checkout of another commit: its renegade_b200 package and library) the two builds run
alternately, each round one child process per build (a process loads one binding and one library), and the verdicts
of the two must be equal.  Each number is the median over the
rounds of the median of `reps` calls after a warm-up call of the same shape; the calls end in a synchronise.  Prints the
card (name, power limit, max SM clock) and one JSON line per row.  Needs a CUDA device."""
import argparse
import hashlib
import json
import os
import random
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NS = (1, 2, 8, 32, 128, 512, 2048, 4096, 16384)
KS = (1, 16, 256, 4096)
Q = 21888242871839275222246405745257275088696311157297823662689037894645226208583


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
    return out[0] if out else "unknown"


def _median_ms(fn, reps):
    fn()  # warm-up of this shape
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        out = fn()
        ts.append(1e3 * (time.perf_counter() - t0))
    return statistics.median(ts), out


def worker(pkg_root, reps, profile):
    """The build under pkg_root in this process: every row's median time and a digest of its verdicts."""
    import numpy as np
    sys.path.insert(0, pkg_root)
    import renegade_b200 as rb
    from renegade_b200 import synth
    from renegade_b200.backend import B200Proof, PlonkKzgSnark, VerifyingKey, pairing_check_many
    srs_head = open(os.path.join(ROOT, "tests", "golden", "srs_head.bin"), "rb").read()
    raw = np.frombuffer(open(os.path.join(ROOT, "tests", "golden", "srs_g2.bin"), "rb").read(), dtype=np.uint64)
    h, tau_h = raw[:16].copy(), raw[16:32].copy()
    ctx = rb.Context(0)
    params = rb.parse_ptau_file(ctx, srs_head, count=512)
    pts = params.powers_of_g_host
    neg = pts.copy()
    for i in range(512):
        y = int.from_bytes(pts[i, 4:8].tobytes(), "little")
        neg[i, 4:8] = np.frombuffer(((Q - y) % Q).to_bytes(32, "little"), dtype="<u8")
    g2 = np.stack([tau_h, h])
    rows = {}
    for n in NS:  # the SRS ratio checks, every 7th with a skipped power (fails)
        g1 = np.stack([np.stack([pts[i % 509], neg[i % 509 + (2 if i % 7 == 3 else 1)]]) for i in range(n)])
        ms, got = _median_ms(lambda: pairing_check_many(ctx, g2, g1), reps)
        rows[f"pair n={n}"] = (ms, hashlib.sha256(np.asarray(got, dtype=np.uint8).tobytes()).hexdigest()[:16])
    circ = synth.synth_circuit(7, num_inputs=4, seed=2, check=True)
    pk = PlonkKzgSnark.preprocess(ctx, params.powers_of_g, 7, 4, circ.selectors, circ.perm, circ.k)
    vk = VerifyingKey.from_proving_key(pk, h, tau_h)
    base = [PlonkKzgSnark.prove_with_link_hint(ctx, pk, circ.wires, circ.pub_inputs, synth.splitmix_blinders(b))[0]
            for b in range(4)]
    for k in KS:
        for frac in (0.0, 0.25):
            bad = set(random.Random(k).sample(range(k), int(round(frac * k)))) if frac else set()
            proofs = []
            for i in range(k):
                p = base[i % len(base)]
                if i in bad:
                    p = B200Proof.from_buffer_copy(bytes(p))
                    p.wires_evals[3][0] ^= 1
                proofs.append(p)
            ms, got = _median_ms(lambda: PlonkKzgSnark.verify_each(ctx, [vk] * k, [circ.pub_inputs] * k, proofs), reps)
            assert got == [i not in bad for i in range(k)]
            rows[f"each k={k} failing={len(bad)}"] = (ms, hashlib.sha256(bytes(got)).hexdigest()[:16])
    kernels = {}
    if profile:  # device time per kernel of small calls, in a pass of its own
        from torch.profiler import ProfilerActivity, profile as prof
        g1 = np.stack([np.stack([pts[i], neg[i + 1]]) for i in range(2)])
        with prof(activities=[ProfilerActivity.CUDA]) as p:
            for _ in range(reps):
                pairing_check_many(ctx, g2, g1[:1])
                PlonkKzgSnark.verify_each(ctx, [vk], [circ.pub_inputs], base[:1])
        for ev in p.key_averages():
            if ev.device_time_total > 0:
                kernels[ev.key[:80]] = {"calls": ev.count, "mean_us": round(ev.device_time_total / max(1, ev.count), 1)}
    pk.free()
    ctx.close()
    return {"rows": rows, "kernels": kernels}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--parent", default=None, help="a built checkout of another commit to run alternately")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    ap.add_argument("--worker", default=None, help=argparse.SUPPRESS)
    ap.add_argument("--profile", action="store_true", help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.worker:
        print(json.dumps(worker(args.worker, args.reps, args.profile)))
        return
    libs = {"change": ROOT}
    if args.parent:
        libs = {"parent": os.path.abspath(args.parent), **libs}
    print(json.dumps({"card": card()}), flush=True)
    runs = {name: [] for name in libs}
    for r in range(args.rounds):
        for name, pkg_root in libs.items():
            env = {k: v for k, v in os.environ.items() if k != "B200_LIB_PATH"}
            cmd = [sys.executable, os.path.abspath(__file__), "--worker", pkg_root, "--reps", str(args.reps)]
            if r == args.rounds - 1:
                cmd.append("--profile")
            out = subprocess.run(cmd, env=env, capture_output=True, text=True, check=True).stdout.strip().splitlines()
            runs[name].append(json.loads(out[-1]))
    table = []
    for key in runs[next(iter(runs))][0]["rows"]:
        row = {"row": key}
        for name in libs:
            row[f"{name}_ms"] = round(statistics.median(run["rows"][key][0] for run in runs[name]), 2)
        digests = {run["rows"][key][1] for name in libs for run in runs[name]}
        row["verdicts_equal"] = len(digests) == 1
        table.append(row)
        print(json.dumps(row), flush=True)
    kernels = {name: runs[name][-1]["kernels"] for name in libs}
    print(json.dumps({"kernels": kernels}), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump({"card": card(), "rows": table, "kernels": kernels}, f, indent=1)


if __name__ == "__main__":
    main()
