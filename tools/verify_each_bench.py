"""Per-item verification against the combined check: b200_plonk_verify_each, b200_plonk_batch_verify with verdicts, and
the host single verifiers, on batches of k proofs (2^7 gates, 4 public inputs, the reference's SRS head) of which a
seeded fraction is tampered; and the checks per second of b200_pairing_check_many against the host b200_pairing_check.

    python tools/verify_each_bench.py [--ks 16,256,4096] [--fails 0,0.01,0.5] [--out FILE.json]

Each row times one call after a warm-up call of the same k (device times: the calls end in a synchronise).  The
host singles are timed on min(k, 64) items and scaled to k.  Every row also checks that the three give the same
verdicts.  Needs a CUDA device."""
import argparse
import json
import os
import random
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import renegade_b200 as rb  # noqa: E402
from renegade_b200 import synth  # noqa: E402
from renegade_b200.backend import (B200Proof, PlonkKzgSnark, VerifyingKey, pairing_check,  # noqa: E402
                                   pairing_check_many)

Q = 21888242871839275222246405745257275088696311157297823662689037894645226208583


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ks", default="16,256,4096")
    ap.add_argument("--fails", default="0,0.01,0.5")
    ap.add_argument("--out", default=None, help="also write the results here (JSON)")
    args = ap.parse_args()
    srs_head = open(os.path.join(ROOT, "tests", "golden", "srs_head.bin"), "rb").read()
    raw = np.frombuffer(open(os.path.join(ROOT, "tests", "golden", "srs_g2.bin"), "rb").read(), dtype=np.uint64)
    h, tau_h = raw[:16].copy(), raw[16:32].copy()
    ctx = rb.Context(0)
    params = rb.parse_ptau_file(ctx, srs_head, count=512)
    srs = params.powers_of_g
    circ = synth.synth_circuit(7, num_inputs=4, seed=2, check=True)
    pk = PlonkKzgSnark.preprocess(ctx, srs, 7, 4, circ.selectors, circ.perm, circ.k)
    vk = VerifyingKey.from_proving_key(pk, h, tau_h)
    base = [PlonkKzgSnark.prove_with_link_hint(ctx, pk, circ.wires, circ.pub_inputs, synth.splitmix_blinders(b))[0]
            for b in range(4)]
    rows = []
    for k in (int(x) for x in args.ks.split(",")):
        for frac in (float(x) for x in args.fails.split(",")):
            bad = set(random.Random(k * 1000 + int(frac * 100)).sample(range(k), int(round(frac * k))))
            proofs = []
            for i in range(k):
                p = base[i % len(base)]
                if i in bad:
                    p = B200Proof.from_buffer_copy(bytes(p))
                    p.wires_evals[3][0] ^= 1
                proofs.append(p)
            vks, pis = [vk] * k, [circ.pub_inputs] * k
            PlonkKzgSnark.verify_each(ctx, vks, pis, proofs)  # warm-up of this shape
            if not bad:
                PlonkKzgSnark.batch_verify(ctx, vks, pis, proofs)
            t0 = time.perf_counter()
            each = PlonkKzgSnark.verify_each(ctx, vks, pis, proofs)
            t1 = time.perf_counter()
            ok, batch = PlonkKzgSnark.batch_verify(ctx, vks, pis, proofs)
            t2 = time.perf_counter()
            ns = min(k, 64)
            single = [PlonkKzgSnark.verify(vk, circ.pub_inputs, p) for p in proofs[:ns]]
            t3 = time.perf_counter()
            want = [i not in bad for i in range(k)]
            row = {"k": k, "failing": len(bad), "verify_each_ms": round(1e3 * (t1 - t0), 2),
                   "batch_verify_ms": round(1e3 * (t2 - t1), 2), "host_singles_ms": round(1e3 * (t3 - t2) * k / ns, 1),
                   "verdicts_agree": each == batch == want and single == want[:ns]}
            rows.append(row)
            print(json.dumps(row), flush=True)
    # pairing checks per second: the SRS ratio checks e(P_i, tau H) e(-P_{i+1}, H)
    pts = params.powers_of_g_host
    neg = pts.copy()
    for i in range(512):
        y = int.from_bytes(pts[i, 4:8].tobytes(), "little")
        neg[i, 4:8] = np.frombuffer(((Q - y) % Q).to_bytes(32, "little"), dtype="<u8")
    g2 = np.stack([tau_h, h])
    pair_rows = []
    for n in (511, 4088):
        g1 = np.stack([np.stack([pts[i % 511], neg[i % 511 + 1]]) for i in range(n)])
        pairing_check_many(ctx, g2, g1)
        t0 = time.perf_counter()
        got = pairing_check_many(ctx, g2, g1)
        dt = time.perf_counter() - t0
        pair_rows.append({"n_checks": n, "device_ms": round(1e3 * dt, 2), "device_checks_per_s": round(n / dt),
                          "all_one": bool(got.all())})
        print(json.dumps(pair_rows[-1]), flush=True)
    t0 = time.perf_counter()
    for i in range(64):
        assert pairing_check([pts[i], neg[i + 1]], [tau_h, h])
    host_rate = 64 / (time.perf_counter() - t0)
    print(json.dumps({"host_checks_per_s": round(host_rate, 1)}), flush=True)
    result = {"card": card(), "verify": rows, "pairing_check_many": pair_rows, "host_checks_per_s": round(host_rate, 1)}
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)
    print(json.dumps({"card": result["card"]}))
    pk.free()
    ctx.close()


if __name__ == "__main__":
    main()
