"""Batch proving (`b200_plonk_prove_batch`) against the prover pool of single proofs, on one GPU.

    python tools/prove_batch_bench.py [--ks 1,4,16,64] [--proofs 128] [--circuits settlement,vbc,validity,synthetic]

For each circuit — the 2^12 private-settlement statement, VALID BALANCE CREATE (2^13), INTENT AND BALANCE VALIDITY (2^14),
all restated in examples/host_circuits, and the 2^16 synthetic circuit of bench.py — it times, with the witness in pinned
host memory and on device-generated known-discrete-log bases:
  * batch calls of k proofs on one context, k in --ks (proofs/s over --proofs proofs, after one warm-up call);
  * batch jobs of 16 proofs on a pool of 2 and of 4 workers;
  * the pool of single proofs with 16 in flight (16 workers), what bench.py's real-statement leg runs;
and checks in the same run that every batch item's bytes equal the single proof's.  It also measures the commitment
epilogue's crossover: batched MSMs of c commitments of 2^12, 2^13 and 2^14 points with the window sums finished on the host
(msm_finish_batch) and on the device (msm_horner_kernel; B200_HOST_HORNER=0, in a child process).  One JSON line per
result, headed by the card's name and power limit.
"""
import argparse
import json
import os
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
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        out = "unknown"
    return name, out


def circuits(names):
    from host_circuits import intent_and_balance_validity as val
    from host_circuits import private_settlement as ps
    from host_circuits import valid_balance_create as vbc
    from renegade_b200 import synth
    out = []
    for nm in names:
        parties, pst = ps.create_witness_statement(1)
        settlement = ps.IntentAndBalancePrivateSettlementCircuit.build(parties, pst)
        if nm == "settlement":
            out.append(("private_settlement", settlement.finalize_for_arithmetization()))
        elif nm == "vbc":
            w, st = vbc.create_witness_statement(1)
            out.append(("valid_balance_create", vbc.ValidBalanceCreate.build(w, st).finalize_for_arithmetization()))
        elif nm == "validity":
            w, st = val.create_witness_statement(seed=70)
            out.append(("intent_and_balance_validity", val.IntentAndBalanceValidityCircuit.build(w, st, settlement.get_circuit_layout()).finalize_for_arithmetization()))
        elif nm == "synthetic":
            out.append(("synthetic_2^16", synth.synth_circuit(16, num_inputs=8, seed=1)))
    return out


def horner_leg(ks):
    """Batched MSMs of c commitments: ms per call with the current B200_HOST_HORNER setting."""
    import ctypes as C
    import torch
    import renegade_b200 as rb
    ctx = rb.Context(0)
    res = {}
    for log_n in (12, 13, 14):
        n = 1 << log_n
        d_srs = torch.empty((n + 3, 8), dtype=torch.int64, device="cuda")
        ctx.known_dlog_bases_device(SEED_SRS, n + 3, d_srs.data_ptr())
        bases = ctx.load_bases_device(d_srs.data_ptr(), n + 3)
        cmax = max(ks)
        d_sc = torch.empty((cmax * n, 4), dtype=torch.int64, device="cuda")
        ctx.splitmix_fr_device(7, cmax * n, d_sc.data_ptr(), True)
        torch.cuda.synchronize()
        for c in ks:
            out = (C.c_uint64 * (8 * c))()
            inf = (C.c_int * c)()
            call = lambda: ctx._lib.b200_msm_batch_device(ctx._h, bases._h, 0, C.c_void_p(d_sc.data_ptr()), n, n, c, 1, out, inf)
            call()
            ts = []
            for _ in range(7):
                t = time.perf_counter()
                assert call() == 0
                ts.append(time.perf_counter() - t)
            res[f"{log_n}:{c}"] = sorted(ts)[3] * 1e3
        bases.free()
    print(json.dumps(res), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ks", default="1,4,16,64")
    ap.add_argument("--proofs", type=int, default=128)
    ap.add_argument("--circuits", default="settlement,vbc,validity,synthetic")
    ap.add_argument("--horner", default="1,2,5,10,20,40,64")  # b200_msm_batch_device takes at most 64
    ap.add_argument("--horner-leg", action="store_true", help=argparse.SUPPRESS)
    args = ap.parse_args()
    horner_ks = [int(x) for x in args.horner.split(",")]
    if args.horner_leg:
        return horner_leg(horner_ks)
    import torch
    import renegade_b200 as rb
    from renegade_b200 import synth
    from renegade_b200.backend import PlonkKzgSnark, ProverPool, prove_raw

    name, power = card()
    print(json.dumps({"card": name, "power_limit": power}), flush=True)
    ks = [int(x) for x in args.ks.split(",")]
    total = args.proofs
    for cname, circ in circuits(args.circuits.split(",")):
        n = circ.n
        d_srs = torch.empty((n + 3, 8), dtype=torch.int64, device="cuda")
        ctx = rb.Context(0)
        ctx.known_dlog_bases_device(SEED_SRS, n + 3, d_srs.data_ptr())
        torch.cuda.synchronize()
        bases = ctx.load_bases_device(d_srs.data_ptr(), n + 3)
        pk = PlonkKzgSnark.preprocess(ctx, bases, circ.log_n, circ.num_inputs, circ.selectors, circ.perm, circ.k)
        h_w = torch.from_numpy(np.ascontiguousarray(circ.wires).view(np.int64)).pin_memory()
        wp = h_w.data_ptr()
        bl = [synth.splitmix_blinders(3000 + i) for i in range(max(ks + [16]))]
        row = {"circuit": cname, "log_n": circ.log_n, "num_inputs": circ.num_inputs}
        # the bytes: every batch item equals its single proof
        singles = [bytes(prove_raw(ctx, pk, wp, circ.pub_inputs, b)) for b in bl]
        kk = max(ks)
        proofs, _, st = PlonkKzgSnark.prove_batch(ctx, pk, [wp] * kk, [circ.pub_inputs] * kk, bl[:kk])
        row["batch_bytes_equal_single"] = st == [0] * kk and [bytes(p) for p in proofs] == singles[:kk]
        # one context: batch calls of k
        for k in ks:
            PlonkKzgSnark.prove_batch(ctx, pk, [wp] * k, [circ.pub_inputs] * k, bl[:k])
            calls = max(1, total // k)
            t = time.perf_counter()
            for _ in range(calls):
                PlonkKzgSnark.prove_batch(ctx, pk, [wp] * k, [circ.pub_inputs] * k, bl[:k])
            row[f"batch_k{k}_proofs_per_s"] = calls * k / (time.perf_counter() - t)
        pk.free()
        bases.free()
        ctx.close()
        # pools: batch jobs of 16 on 2 and 4 workers; single proofs with 16 in flight
        for workers, kind in ((2, "batch16"), (4, "batch16"), (16, "single")):
            pool = ProverPool(0, workers=workers)
            pc = pool.context(0)
            b2 = pc.load_bases_device(d_srs.data_ptr(), n + 3)
            pk2 = PlonkKzgSnark.preprocess(pc, b2, circ.log_n, circ.num_inputs, circ.selectors, circ.perm, circ.k)

            def run(count):
                if kind == "single":
                    tks = [pool.submit_prove(pk2, wp, circ.pub_inputs, bl[i % 16]) for i in range(count)]
                else:
                    tks = [pool.submit_prove_batch(pk2, [wp] * 16, [circ.pub_inputs] * 16, bl[:16]) for _ in range(count // 16)]
                for tk in tks:
                    pool.wait(tk)
            run(max(2 * 16 * workers, 32))  # every worker sized (and, for single proofs, its graphs captured)
            t = time.perf_counter()
            run(total)
            row[f"pool{workers}_{kind}_proofs_per_s"] = (total // 16 * 16 if kind != "single" else total) / (time.perf_counter() - t)
            pk2.free()
            b2.free()
            pool.close()
        print(json.dumps(row), flush=True)
        del d_srs
        torch.cuda.empty_cache()
    # commitment epilogue: host vs device Horner, same calls
    for env, label in (({}, "host_horner_ms"), ({"B200_HOST_HORNER": "0"}, "device_horner_ms")):
        r = subprocess.run([sys.executable, os.path.abspath(__file__), "--horner-leg", "--horner", args.horner],
                           env={**os.environ, **env}, capture_output=True, text=True, timeout=900)
        line = [x for x in r.stdout.splitlines() if x.startswith("{")]
        print(json.dumps({label: json.loads(line[-1]) if line else r.stderr[-500:]}), flush=True)


if __name__ == "__main__":
    main()
