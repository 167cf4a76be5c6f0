"""Batch link proving (`b200_plonk_link_batch`) against single link proofs, on one GPU.

    python tools/link_batch_bench.py [--items 1024] [--reps 5]

Two workloads, on device-generated known-discrete-log bases of 2^16 + 3 points:
  * private_match: the four link proofs of one private match (two INTENT AND BALANCE VALIDITY and two OUTPUT BALANCE
    VALIDITY hints against the PRIVATE SETTLEMENT hint, N = 2^15 and 2^14), from the statements restated in
    examples/host_circuits, proved on the same bases;
  * synthetic_2^16: one pair of 2^16 + 2 coefficients (N = 2^17) that agree on a group of 8 roots.
For each it times, over --items link proofs cycling through the workload's pairs (host arrays, as the pool's bundles
hand them over):
  * single b200_plonk_link calls on one context (graph replay);
  * batch calls of k = 4, 16, 64 on one context;
  * a pool of 16 workers with every single link job in flight;
  * batch jobs of 4 and of 16 on a pool of 4 workers;
and checks in the same run that every batch item's bytes equal the single call's.  It also prints the wall time of one
private match's five proofs and of its four link proofs, each run one after the other on an idle context (every call
waits for its own GPU work), so the share the links take is measured.  One JSON line per result, headed by the card's
name and power limit.
"""
import argparse
import json
import os
import random
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "examples"))

import numpy as np  # noqa: E402

SEED_SRS = 0x5EED
R = 0x30644E72E131A029B85045B68181585D2833E84879B97091_43E1F593F0000001
MONT = 1 << 256


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


def to_mont(vals):
    raw = b"".join((v * MONT % R).to_bytes(32, "little") for v in vals)
    return np.frombuffer(raw, dtype=np.uint64).reshape(-1, 4).copy()


def hint(ctx, bases, m):
    from renegade_b200.backend import LinkingHint
    xy, inf = ctx.msm(bases, m, montgomery=True)
    return LinkingHint(m, np.zeros(8, dtype=np.uint64) if inf else xy)


def synthetic_pair(ctx, bases, log_len=16, alignment=10, offset=100, size=8):
    """a1 = a2 + Z_D q, len 2^log_len + 2 each"""
    from renegade_b200.backend import GroupLayout
    rng = random.Random(0x11)
    g_limbs = ctx.domain_generator(alignment).reshape(-1)
    g = int.from_bytes(g_limbs.tobytes(), "little") * pow(MONT, -1, R) % R
    z = [1]
    for i in range(size):
        r = pow(g, offset + i, R)
        z = [((z[j - 1] if j else 0) - r * (z[j] if j < len(z) else 0)) % R for j in range(len(z) + 1)]
    n = (1 << log_len) + 2
    q = [rng.randrange(R) for _ in range(n - size)]
    delta = [0] * n
    for i, zi in enumerate(z):
        for j, qj in enumerate(q):
            delta[i + j] = (delta[i + j] + zi * qj) % R
    a2 = [rng.randrange(R) for _ in range(n)]
    a1 = [(x + d) % R for x, d in zip(a2, delta)]
    return hint(ctx, bases, to_mont(a1)), hint(ctx, bases, to_mont(a2)), GroupLayout(alignment, offset, size)


def private_match(ctx, bases, reps):
    """the four link triples of one private match, and the wall ms of its five proofs and of its four link proofs"""
    from host_circuits import intent_and_balance_validity as val
    from host_circuits import output_balance_validity as obv
    from host_circuits import private_settlement as ps
    from host_circuits import statements as st
    from renegade_b200 import circuit_types as ct
    from renegade_b200 import synth
    from renegade_b200.backend import GroupLayout, PlonkKzgSnark, link_proofs
    g2 = np.frombuffer(open(os.path.join(ROOT, "tests", "golden", "srs_g2.bin"), "rb").read(), dtype=np.uint64)
    ct.set_system_srs(ctx, bases, g2[:16].copy(), g2[16:32].copy())
    parties, _ = ps.create_witness_statement(seed=61)
    validity = [val.create_witness_statement(seed=70 + i, intent=parties[i].intent, balance=parties[i].input_balance)
                for i in (0, 1)]
    out_validity = [obv.create_witness_statement(80 + i, parties[i].output_balance) for i in (0, 1)]
    parties, statement = ps.create_witness_statement(
        seed=61, linked=[(validity[i][0].new_amount_public_share, validity[i][0].post_match_balance_shares,
                          out_validity[i][0].post_match_balance_shares) for i in (0, 1)])
    S = st.IntentAndBalancePrivateSettlementCircuit
    jobs = [(S, parties, statement, None)]
    for i in (0, 1):
        jobs.append((st.IntentAndBalanceValidityCircuit, *validity[i], ps.PARTY_LINKS[i]))
        jobs.append((st.OutputBalanceValidityCircuit, *out_validity[i], ps.OUTPUT_LINKS[i]))
    arith = [C._arithmetize(w, s) for C, w, s, _ in jobs]
    bl = synth.splitmix_blinders(5)
    hints = [PlonkKzgSnark.prove_with_link_hint(ctx, pk, c.wires, c.pub_inputs, bl)[1] for pk, c in arith]
    layouts = S.get_circuit_layout()
    triples = [(hints[j], hints[0], GroupLayout(layouts[gid].alignment, layouts[gid].offset, layouts[gid].size))
               for j, (_, _, _, gid) in enumerate(jobs) if gid is not None]

    def wall(fn):
        fn()  # eager / capture
        fn()
        ts = []
        for _ in range(reps):
            t = time.perf_counter()
            fn()
            ts.append(time.perf_counter() - t)
        return sorted(ts)[len(ts) // 2] * 1e3

    proofs_ms = wall(lambda: [PlonkKzgSnark.prove_with_link_hint(ctx, pk, c.wires, c.pub_inputs, bl) for pk, c in arith])
    links_ms = wall(lambda: [link_proofs(ctx, bases, *t) for t in triples])
    sizes = [[int(c.log_n) for _, c in arith], [int(t[0].linking_wire_poly.shape[0]) for t in triples]]
    return triples, proofs_ms, links_ms, sizes


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--items", type=int, default=1024)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    import torch
    import renegade_b200 as rb
    from renegade_b200.backend import ProverPool, link_proofs, link_proofs_batch

    name, power = card()
    print(json.dumps({"card": name, "power_limit": power}), flush=True)
    n = (1 << 16) + 3
    d_srs = torch.empty((n, 8), dtype=torch.int64, device="cuda")
    ctx = rb.Context(0)
    ctx.known_dlog_bases_device(SEED_SRS, n, d_srs.data_ptr())
    torch.cuda.synchronize()
    bases = ctx.load_bases_device(d_srs.data_ptr(), n)
    pm, proofs_ms, links_ms, sizes = private_match(ctx, bases, args.reps)
    batch_ms = []
    for _ in range(args.reps + 1):
        t = time.perf_counter()
        link_proofs_batch(ctx, bases, pm)
        batch_ms.append((time.perf_counter() - t) * 1e3)
    print(json.dumps({"private_match_bundle": {
        "proof_log_n": sizes[0], "link_hint_lengths": sizes[1],
        "five_proofs_ms": proofs_ms, "four_single_links_ms": links_ms, "four_links_as_one_batch_ms": sorted(batch_ms[1:])[args.reps // 2],
        "link_share_of_bundle": links_ms / (links_ms + proofs_ms)}}), flush=True)
    workloads = [("private_match", pm), ("synthetic_2^16", [synthetic_pair(ctx, bases)])]
    total = args.items
    for wname, base in workloads:
        items = [base[i % len(base)] for i in range(total)]
        row = {"workload": wname, "items": total}
        singles = [bytes(link_proofs(ctx, bases, *t)[0]) for t in base]  # eager; the next call captures
        for t in base:
            link_proofs(ctx, bases, *t)
        want = [singles[i % len(base)] for i in range(total)]
        proofs, _, st = link_proofs_batch(ctx, bases, items)
        row["batch_bytes_equal_single"] = st == [0] * total and [bytes(p) for p in proofs] == want
        t = time.perf_counter()
        for it in items:
            link_proofs(ctx, bases, *it)
        row["single_links_per_s"] = total / (time.perf_counter() - t)
        for k in (4, 16, 64):
            link_proofs_batch(ctx, bases, items[:k])
            calls = max(1, total // k)
            t = time.perf_counter()
            for c in range(calls):
                link_proofs_batch(ctx, bases, items[c * k % total:][:k] if total >= k else items[:k])
            row[f"batch_k{k}_links_per_s"] = calls * k / (time.perf_counter() - t)
        for workers, kind in ((16, "single"), (4, "batch4"), (4, "batch16")):
            pool = ProverPool(0, workers=workers)
            pc = pool.context(0)
            b2 = pc.load_bases_device(d_srs.data_ptr(), n)
            ok = True

            def run(count):
                nonlocal ok
                if kind == "single":
                    tks = [pool.submit_link(b2, *items[i % total]) for i in range(count)]
                    got = [bytes(pool.wait(tk)) for tk in tks]
                else:
                    k = int(kind[5:])
                    tks = [pool.submit_link_batch(b2, [items[(j * k + i) % total] for i in range(k)]) for j in range(count // k)]
                    got = [bytes(p) for tk in tks for p in pool.wait(tk)[0]]
                ok = ok and got == [want[i % total] for i in range(len(got))]
            run(max(4 * workers, 32))  # every worker sized, its graphs captured
            t = time.perf_counter()
            run(total)
            done = total if kind == "single" else total // int(kind[5:]) * int(kind[5:])
            row[f"pool{workers}_{kind}_links_per_s"] = done / (time.perf_counter() - t)
            row[f"pool{workers}_{kind}_bytes_equal_single"] = ok
            b2.free()
            pool.close()
        print(json.dumps(row), flush=True)
    from renegade_b200 import circuit_types as ct
    ct.clear_key_cache()
    bases.free()
    ctx.close()


if __name__ == "__main__":
    main()
