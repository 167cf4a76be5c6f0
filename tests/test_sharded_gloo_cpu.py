"""world_size-2 gloo test (CPU) of the multi-GPU MSM's host-visible logic: the library's shard partition
(`b200_shard_range`), one gather of the per-rank partials and their combination (`b200_g1_sum_affine`).
On the CPU box the per-rank partial is produced by the oracle (test infrastructure) and the gather runs over
gloo; on GPUs the partials come from the CUDA path and travel through `ncclAllGather` inside the library
(`b200_multi_msm`, tests/test_gpu_multi.py).  The host combine itself is held to a Python-integer affine sum on its
edge cases: no records, identity flags, doubling, cancellation, and an off-curve record (not checked, recorded)."""
import os
import sys

import numpy as np
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _worker(rank, world, port, n, q):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "oracle"))
    import torch.distributed as dist
    import oracle_c
    from renegade_b200.sharded import combine_partials, shard_range
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        b, e = shard_range(n, rank, world)
        bases = oracle_c.known_dlog_bases(0xB200, e - b, first=b)
        scalars = oracle_c.splitmix_fr(0x5CA1A8, e - b, False, first=b)
        xy, inf = oracle_c.msm(bases, scalars)
        mine = np.zeros(9, dtype=np.uint64)
        mine[:8] = xy
        mine[8] = 1 if inf else 0
        gathered = [None] * world
        dist.all_gather_object(gathered, mine.tolist())
        out, oinf = combine_partials(np.array(gathered, dtype=np.uint64))
        q.put((rank, out.tolist(), oinf))
    finally:
        dist.destroy_process_group()


def test_sharded_msm_two_ranks(oracle):
    n, world, port = 301, 2, 29731
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, world, port, n, q)) for r in range(world)]
    for p in procs:
        p.start()
    results = [q.get(timeout=120) for _ in range(world)]
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    full, finf = oracle.msm(oracle.known_dlog_bases(0xB200, n), oracle.splitmix_fr(0x5CA1A8, n, False))
    for rank, out, oinf in results:
        assert not oinf and (np.array(out, dtype=np.uint64) == full).all(), rank


def _records(py, points, flags=None):
    """(k, 9) records x || y (Montgomery) || identity flag of affine points given as Python integers (None: the
    identity, encoded as zeros and flagged)."""
    rec = np.zeros((len(points), 9), dtype=np.uint64)
    for i, p in enumerate(points):
        rec[i, :8] = np.frombuffer(py.encode_g1_mont(p), dtype=np.uint64)
        rec[i, 8] = 1 if p is None else 0
    if flags is not None:
        rec[:, 8] = flags
    return rec


def _affine_sum(py, points, flags):
    acc = None
    for p, f in zip(points, flags):
        if not f:
            acc = py.g1_add(acc, p)
    return acc


def _combined(py, rec):
    from renegade_b200.sharded import combine_partials
    out, inf = combine_partials(rec)
    if inf:
        assert not out.any()
        return None
    return py.decode_g1_mont(out.tobytes(), 0)


def _seeded_points(oracle, py, seed, k):
    raw = oracle.known_dlog_bases(seed, k).tobytes()
    return [py.decode_g1_mont(raw, i) for i in range(k)]


def test_combine_partials_edge_cases(oracle, pyoracle):
    """`combine_partials` (`b200_g1_sum_affine`, the host combine for callers that gather the partials themselves) =
    the Python-integer affine sum of the records not flagged as the identity: no records, every record flagged, P + P,
    P + (-P), P + P + (-P), a flagged record holding a real point (ignored), a running sum that doubles, cancels to
    the identity and starts again, and 64 seeded partials with and without flags."""
    py = pyoracle
    P, Q, S = _seeded_points(oracle, py, 0xC0DE, 3)
    nP = py.g1_neg(P)
    two_p = py.g1_add(P, P)
    cases = {
        "k = 0": ([], []),
        "all flagged": ([P, Q, S], [1, 1, 1]),
        "P, P": ([P, P], [0, 0]),
        "P, -P": ([P, nP], [0, 0]),
        "P, P, -P": ([P, P, nP], [0, 0, 0]),
        "flag on a real point": ([P, Q, S], [0, 1, 0]),
        "flag on the first": ([Q, P, S], [1, 0, 0]),
        "identity records": ([None, P, None, P], None),
        "running sum doubles, cancels, restarts": ([P, P, py.g1_neg(two_p), Q, Q, S], [0] * 6),
    }
    pts64 = _seeded_points(oracle, py, 0x64, 64)
    rng = np.random.default_rng(64)
    cases["64 partials"] = (pts64, [0] * 64)
    cases["64 partials, seeded flags"] = (pts64, [int(v) for v in rng.integers(0, 2, 64)])
    for name, (pts, flags) in cases.items():
        flags = [1 if p is None else 0 for p in pts] if flags is None else flags
        exp = _affine_sum(py, pts, flags)
        assert _combined(py, _records(py, pts, flags)) == exp, name
    # preconditions of the named cases
    assert _affine_sum(py, [P, nP], [0, 0]) is None and _affine_sum(py, [P, P, py.g1_neg(two_p)], [0] * 3) is None
    assert _combined(py, _records(py, [P, P], [0, 0])) == py.g1_mul(P, 2)


def test_combine_partials_does_not_check_the_curve(oracle, pyoracle):
    """Recorded behaviour: records are not checked against the curve.  An off-curve record (y + 1) is added by the
    chord formula like any other point, first or last, and the call succeeds with a result off the curve."""
    py = pyoracle
    P, Q = _seeded_points(oracle, py, 0xBAD, 2)
    off = (Q[0], (Q[1] + 1) % py.Q)
    assert not py.g1_is_on_curve(off)
    chord = py.g1_add(P, off)  # the affine chord formula, which never reads the curve constant
    assert chord is not None and not py.g1_is_on_curve(chord)
    assert _combined(py, _records(py, [P, off], [0, 0])) == chord
    assert _combined(py, _records(py, [off, P], [0, 0])) == chord
    assert _combined(py, _records(py, [off], [0])) == off
    assert _combined(py, _records(py, [off], [1])) is None


def test_shard_range_is_a_partition():
    from renegade_b200.sharded import shard_range
    for n in (0, 1, 7, 8, 301, 1 << 20, (1 << 24) + 3):
        for world in (1, 2, 3, 4, 8):
            cuts = [shard_range(n, r, world) for r in range(world)]
            assert cuts[0][0] == 0 and cuts[-1][1] == n
            assert all(cuts[i][1] == cuts[i + 1][0] for i in range(world - 1))
            sizes = [e - b for b, e in cuts]
            assert max(sizes) - min(sizes) <= 1 and sizes == sorted(sizes, reverse=True)
