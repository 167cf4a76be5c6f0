"""Kernel and graph launches per call, and a digest of every result, for a fixed set of seeded calls on one GPU.

    python tools/launch_parity.py [--root DIR] > launches.json

Run it on two builds of the library (--root: the tree whose renegade_b200 package is imported, by default this one)
and diff the two outputs: a change that is meant to keep what the library launches and computes must print the same
JSON object.  The calls, each counted on its own (b200_kernel_launches, b200_graph_launches):
  * a single proof at 2^16 three times on one context: eager, captured as CUDA graphs, replayed;
  * b200_plonk_prove_batch at k = 3 and k = 12, on each side of the batch prover's device-Horner crossover;
  * b200_plonk_link_batch at k = 3 and k = 12, and a single link proof twice (eager, then through its graphs);
  * a context MSM at 2^16, and b200_multi_msm at 2^20 from device and from host scalars.
"""
import argparse
import hashlib
import json
import os
import random
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
R = 0x30644E72E131A029B85045B68181585D2833E84879B97091_43E1F593F0000001
MONT = 1 << 256


def digest(*parts) -> str:
    h = hashlib.sha256()
    for p in parts:
        h.update(bytes(p))
    return h.hexdigest()[:32]


def to_mont(vals):
    import numpy as np
    raw = b"".join((v * MONT % R).to_bytes(32, "little") for v in vals)
    return np.frombuffer(raw, dtype=np.uint64).reshape(-1, 4).copy()


def link_triple(ctx, bases, seed, log_len=12, alignment=10, offset=100, size=8):
    """(hint_a, hint_b, layout) with a1 = a2 + Z_D q: the two polynomials agree on the group's roots"""
    import numpy as np
    from renegade_b200.backend import GroupLayout, LinkingHint
    rng = random.Random(seed)
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
    hints = []
    for a in (a1, a2):
        m = to_mont(a)
        xy, inf = ctx.msm(bases, m, montgomery=True)
        hints.append(LinkingHint(m, np.zeros(8, dtype=np.uint64) if inf else xy))
    return hints[0], hints[1], GroupLayout(alignment, offset, size)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--root", default=ROOT)
    args = ap.parse_args()
    sys.path.insert(0, os.path.abspath(args.root))
    import numpy as np
    import torch
    import renegade_b200 as rb
    from renegade_b200 import synth
    from renegade_b200.backend import PlonkKzgSnark, link_proofs, link_proofs_batch
    from renegade_b200.sharded import MultiGpu

    out = {}
    ctx = rb.Context(0)

    def counted(name, fn, result_bytes):
        k0, g0 = ctx.kernel_launches(), ctx.graph_launches()
        res = fn()
        out[name] = {"kernels": ctx.kernel_launches() - k0, "graphs": ctx.graph_launches() - g0,
                     "digest": digest(*result_bytes(res))}
        return res

    log_n = 16
    n = 1 << log_n
    d_srs = torch.empty((n + 3, 8), dtype=torch.int64, device="cuda:0")
    torch.cuda.synchronize()
    ctx.known_dlog_bases_device(0x5EED, n + 3, d_srs.data_ptr())
    srs = ctx.load_bases_device(d_srs.data_ptr(), n + 3)
    circ = synth.synth_circuit(log_n, num_inputs=8, seed=0xC1C)
    pk = PlonkKzgSnark.preprocess(ctx, srs, log_n, circ.num_inputs, circ.selectors, circ.perm, circ.k)
    bl = [synth.splitmix_blinders(100 + i) for i in range(16)]

    def proof_bytes(r):
        return [bytes(r[0]), r[1].linking_wire_poly.tobytes()]
    ctx.use_graphs(True)
    for i, label in enumerate(("eager", "capture", "replay")):
        counted(f"prove_2^16_{label}", lambda: PlonkKzgSnark.prove_with_link_hint(ctx, pk, circ.wires, circ.pub_inputs, bl[i]),
                proof_bytes)
    for k in (3, 12):
        counted(f"prove_batch_k{k}",
                lambda: PlonkKzgSnark.prove_batch(ctx, pk, [circ.wires] * k, [circ.pub_inputs] * k, bl[:k], link_hints=True),
                lambda r: [bytes(p) for p in r[0]] + [h.linking_wire_poly.tobytes() for h in r[1]] + [bytes(np.array(r[2]))])

    triples = [link_triple(ctx, srs, 0x11 + i) for i in range(3)]
    for k in (3, 12):
        counted(f"link_batch_k{k}", lambda: link_proofs_batch(ctx, srs, [triples[i % 3] for i in range(k)]),
                lambda r: [bytes(p) for p in r[0]] + [e.tobytes() for e in r[1]] + [bytes(np.array(r[2]))])
    for label in ("eager", "replay"):
        counted(f"link_single_{label}", lambda: link_proofs(ctx, srs, *triples[0]), lambda r: [bytes(r[0]), r[1].tobytes()])

    s16 = np.random.default_rng(7).integers(0, 1 << 64, size=(n, 4), dtype=np.uint64)
    s16[:, 3] &= 0x0FFFFFFFFFFFFFFF  # below r
    counted("msm_2^16", lambda: ctx.msm(srs, s16), lambda r: [r[0].tobytes(), bytes([r[1]])])

    nm = 1 << 20
    multi = MultiGpu.single_process([0])
    mctx = multi.ctx(0)
    mb = multi.known_dlog_bases(0xB200, nm)
    d_sc = torch.empty((nm, 4), dtype=torch.int64, device="cuda:0")
    torch.cuda.synchronize()
    mctx.splitmix_fr_device(0x5CA1A8, nm, d_sc.data_ptr(), montgomery=False)
    h_sc = d_sc.cpu().numpy().view(np.uint64)
    torch.cuda.synchronize()
    for label, fn in (("device", lambda: multi.msm_local(mb, [d_sc.data_ptr()], on_device=True)),
                      ("host", lambda: multi.msm(mb, h_sc))):
        k0, g0 = mctx.kernel_launches(), mctx.graph_launches()
        r = fn()
        out[f"multi_msm_2^20_{label}"] = {"kernels": mctx.kernel_launches() - k0, "graphs": mctx.graph_launches() - g0,
                                          "digest": digest(r[0].tobytes(), bytes([r[1]]))}
    mb.free()
    multi.close()
    ctx.close()
    print(json.dumps(out, sort_keys=True, indent=1))


if __name__ == "__main__":
    main()
