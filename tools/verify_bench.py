"""Batch verification vs the single verifiers, on one GPU.

    python tools/verify_bench.py [--sizes 1,16,256,4096] [--reps 3]

Items: device proofs of synthetic 2^12, 2^13 and 2^14 circuits with 24, 48 and 96 public inputs, plus link proofs
between them, repeated up to each batch size k.  For every k it times
  * the host single verifiers (`b200_plonk_verify` / `b200_plonk_verify_link`) over the k items, one after another;
  * one `b200_plonk_batch_verify` call over the same items (wall clock: the call synchronises), best of --reps;
and checks in the same run that the batch verdicts equal the single verdicts.  It also times one 2-pair
`b200_pairing_check` alone, so the pairing's share of a batch is visible.  Prints one JSON line per k, headed by the
card's name and power limit.
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))

import numpy as np  # noqa: E402

TAU = 0x2B7E151628AED2A6ABF7158809CF4F3C762E7160F38B4DA56A784D9045190CFE
LAYOUT = (10, 100, 16)  # alignment, offset, size of the link group
SHAPES = ((12, 24, 1), (13, 48, 2), (14, 96, 3))  # log_n, num_inputs, seed


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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="1,16,256,4096")
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    import bn254_pairing_py as pr
    import bn254_py as py
    import oracle_c
    import renegade_b200 as rb
    from renegade_b200 import synth
    from renegade_b200.backend import GroupLayout, PlonkKzgSnark, VerifyingKey, link_proofs, pairing_check, verify_link_proof

    name, power = card()
    print(json.dumps({"card": name, "power_limit": power}), flush=True)
    ctx = rb.Context(0)
    tau = oracle_c.int_to_limbs(py.to_mont(TAU % py.R, py.R))
    srs = ctx.load_bases(oracle_c.srs_from_tau(tau, (1 << 14) + 3))
    # h: the G2 generator record of the reference's SRS (tests/golden/srs_g2.bin); tau h for the seeded tau
    raw = open(os.path.join(ROOT, "tests", "golden", "srs_g2.bin"), "rb").read()
    h = np.frombuffer(raw[:128], dtype=np.uint64).copy()
    tau_h = np.frombuffer(pr.encode_g2_mont(pr.g2_mul(pr.decode_g2_mont(raw, 0), TAU % pr.R)), dtype=np.uint64).copy()
    lay = GroupLayout(*LAYOUT)
    vals = [(i * 0x9E3779B9 + 7) % py.R for i in range(lay.size)]
    proofs, hints = [], []  # (vk, pub_inputs, proof)
    for log_n, ni, seed in SHAPES:
        circ = synth.synth_circuit(log_n, num_inputs=ni, seed=seed, check=False, link=(lay.alignment, lay.offset, vals))
        pk = PlonkKzgSnark.preprocess(ctx, srs, log_n, ni, circ.selectors, circ.perm, circ.k)
        vk = VerifyingKey.from_proving_key(pk, h, tau_h)
        for b in range(2):
            proof, hint = PlonkKzgSnark.prove_with_link_hint(ctx, pk, circ.wires, circ.pub_inputs,
                                                             synth.splitmix_blinders(100 * seed + b))
            proofs.append((vk, circ.pub_inputs, proof))
            hints.append(hint)
    links = []
    for a, b in ((0, 2), (2, 4), (1, 5)):
        lp, _ = link_proofs(ctx, srs, hints[a], hints[b], lay)
        links.append((hints[a].linking_wire_comm, hints[b].linking_wire_comm, lp, lay))

    # one 2-pair pairing alone: e(G, tau h) e(-G, tau h)
    g = np.frombuffer(py.encode_g1_mont((1, 2)), dtype=np.uint64)
    ng = np.frombuffer(py.encode_g1_mont(py.g1_neg((1, 2))), dtype=np.uint64)
    t = []
    for _ in range(5):
        t0 = time.perf_counter()
        assert pairing_check([g, ng], [tau_h, tau_h])
        t.append(time.perf_counter() - t0)
    pairing_ms = min(t) * 1e3
    print(json.dumps({"pairing_2pair_ms": round(pairing_ms, 3)}), flush=True)

    for k in [int(x) for x in args.sizes.split(",")]:
        # 3 proofs per link, repeated: proofs first, then links (the batch's item order)
        n_links = k // 4
        n_proofs = k - n_links
        its = [proofs[i % len(proofs)] for i in range(n_proofs)]
        lks = [links[i % len(links)] for i in range(n_links)]
        t0 = time.perf_counter()
        single = [PlonkKzgSnark.verify(vk, pi, p) for vk, pi, p in its]
        single += [verify_link_proof(a, b, lp, l, h, tau_h) for a, b, lp, l in lks]
        single_ms = (time.perf_counter() - t0) * 1e3
        best = None
        for _ in range(args.reps):
            t0 = time.perf_counter()
            ok, verdicts = PlonkKzgSnark.batch_verify(ctx, [i[0] for i in its], [i[1] for i in its], [i[2] for i in its],
                                                      lks, g2=(h, tau_h))
            dt = (time.perf_counter() - t0) * 1e3
            best = dt if best is None else min(best, dt)
        print(json.dumps({"k": k, "proofs": n_proofs, "links": n_links, "single_ms": round(single_ms, 2),
                          "single_per_item_ms": round(single_ms / k, 3), "batch_ms": round(best, 2),
                          "batch_per_item_ms": round(best / k, 4), "speedup": round(single_ms / best, 1),
                          "all_accepted": ok, "verdicts_match": verdicts == single and all(single)}), flush=True)
        assert verdicts == single and ok
    ctx.close()


if __name__ == "__main__":
    main()
