"""Test infrastructure: the workload of tests/test_gpu_bench_regime.py that has to run in a process of its own.

The MSM's and the prover's process-wide switches (B200_QUAD_ADD, B200_TREE_FANIN_LOG, B200_HOST_HORNER, B200_GRAPHS) are
read once per process, and CUDA_DEVICE_MAX_CONNECTIONS only counts when it is set before CUDA starts, so each setting
gets a fresh interpreter:

  python tests/regime_driver.py INPUTS.npz switches   MSMs of every reduction shape, proofs eager and replayed, a batch
  python tests/regime_driver.py INPUTS.npz pool16     bench.py's headline: a pool of 16 workers at 2^16, timing on

INPUTS.npz is written by the test (SRS, circuits, blinders, scalars).  The driver computes and prints ONE JSON line of
hex outputs; the test compares them with the oracle and with its own reference proofs.  It checks nothing itself."""
import ctypes as C
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def hexs(a) -> str:
    return np.ascontiguousarray(a).tobytes().hex()


def circuit(inp, key):
    return {f: inp[f"{key}_{f}"] for f in ("selectors", "perm", "k", "wires", "pub_inputs")}


def preprocess(ctx, bases, c):
    from renegade_b200.backend import PlonkKzgSnark
    log_n = c["wires"].shape[1].bit_length() - 1
    return PlonkKzgSnark.preprocess(ctx, bases, log_n, c["pub_inputs"].shape[0], c["selectors"], c["perm"], c["k"])


def msm_batch(ctx, bases, vectors):
    """b200_msm_batch_device over (batch, n, 4) canonical scalars, 8 elements of padding between vectors"""
    import torch
    from renegade_b200 import _lib
    batch, n = vectors.shape[0], vectors.shape[1]
    stride = n + 8
    s = np.zeros((batch, stride, 4), dtype=np.uint64)
    s[:, :n] = vectors
    t = torch.from_numpy(s.view(np.int64)).cuda()
    torch.cuda.synchronize()
    out = np.zeros((batch, 8), dtype=np.uint64)
    inf = (C.c_int * batch)()
    _lib.check(ctx._lib.b200_msm_batch_device(ctx._h, bases._h, 0, C.c_void_p(t.data_ptr()), n, stride, batch, 0,
                                              out.ctypes.data_as(C.c_void_p), inf))
    return [[hexs(out[i]), bool(inf[i])] for i in range(batch)]


def switches(inp) -> dict:
    import renegade_b200 as rb
    from renegade_b200.backend import PlonkKzgSnark
    ctx = rb.Context(0)
    srs, scalars = inp["srs"], inp["scalars"]
    res = {"plans": {}, "msm": {}, "proofs": {}}

    def lone(name, n, window_bits, pts=None, s=None):
        bases = ctx.load_bases(srs[:n] if pts is None else pts, window_bits=window_bits)
        res["plans"][name] = bases.plan
        out, inf = ctx.msm(bases, scalars[:n] if s is None else s)
        res["msm"][name] = [hexs(out), inf]
        return bases

    for lg in (12, 14, 16):  # latency plans: the short-chain reduction of one MSM alone
        lone(f"latency_2^{lg}", 1 << lg, 1)
    lone("throughput_2^16", 1 << 16, 0)
    # one base repeated, scalars 1 + 8 i (and alternating signs, and two halves): equal and opposite partial sums at every
    # level of the reduction, the P = 0 branches of the four-lane additions included
    one = np.repeat(srs[:1], 256, axis=0)
    for wb in (1, 0):
        for v in ("same", "alt", "wide"):
            lone(f"one_base_{v}_w{wb}", 256, wb, pts=one, s=inp[f"one_base_{v}"])
    lat12 = ctx.load_bases(srs[:1 << 12], window_bits=1)
    res["plans"]["batch"] = lat12.plan
    for b in (5, 12):
        res["msm"][f"batch_{b}"] = msm_batch(ctx, lat12, inp["batch_scalars"][:b])
    bases = ctx.load_bases(srs)
    bl = inp["blinders"]
    for key in ("settlement", "synthetic"):
        c = circuit(inp, key)
        pk = preprocess(ctx, bases, c)
        # eager, captured, replayed (unless B200_GRAPHS=0)
        res["proofs"][key] = [[b, bytes(PlonkKzgSnark.prove_with_link_hint(ctx, pk, c["wires"], c["pub_inputs"], bl[b])[0]).hex()]
                              for b in (0, 1, 2)]
        if key == "settlement":
            proofs, _, st = PlonkKzgSnark.prove_batch(ctx, pk, [c["wires"]] * 2, [c["pub_inputs"]] * 2, [bl[3], bl[4]])
            res["proofs"]["settlement_batch"] = [[b, bytes(p).hex()] for b, p in zip((3, 4), proofs)]
            res["batch_statuses"] = st
        pk.free()
    ctx.close()
    return res


def pool16(inp) -> dict:
    import torch
    from renegade_b200.backend import ProverPool
    n = 1 << 16
    pool = ProverPool(0, workers=16)
    try:
        ctxs = [pool.context(i) for i in range(16)]
        ctx = ctxs[0]
        d_srs = torch.empty((n + 3, 8), dtype=torch.int64, device="cuda")
        torch.cuda.synchronize()
        ctx.known_dlog_bases_device(int(inp["seed_srs"]), n + 3, d_srs.data_ptr())
        srs = ctx.load_bases_device(d_srs.data_ptr(), n + 3)
        c = circuit(inp, "synthetic")
        pk = preprocess(ctx, srs, c)
        h_w = torch.from_numpy(c["wires"].view(np.int64)).pin_memory()
        d_w = h_w.to("cuda")
        torch.cuda.synchronize()
        for x in ctxs:
            x.msm_timing(True)
        bl = inp["blinders"]
        jobs = []  # (blinder index, ticket): three waves from device memory, one from pinned host memory
        for wave in range(4):
            ptr = d_w.data_ptr() if wave < 3 else h_w.data_ptr()
            jobs += [(b, pool.submit_prove(pk, ptr, c["pub_inputs"], bl[b])) for b in ((wave * 16 + j) % len(bl) for j in range(16))]
        out = [[b, bytes(pool.wait(t)).hex()] for b, t in reversed(jobs)]
        launches = sum(x.msm_timing_totals()["launches"] for x in ctxs)
        pk.free()
        srs.free()
        return {"proofs": {"synthetic": out}, "msm_launches": launches,
                "cuda_device_max_connections": os.environ.get("CUDA_DEVICE_MAX_CONNECTIONS")}
    finally:
        pool.close()


if __name__ == "__main__":
    data = dict(np.load(sys.argv[1]))
    print(json.dumps({"switches": switches, "pool16": pool16}[sys.argv[2]](data)), flush=True)
