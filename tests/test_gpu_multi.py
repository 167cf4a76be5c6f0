"""GPU parity of the multi-GPU layer behind the C ABI (`b200_multi_*`, csrc/multi.cu): one MSM sharded by point
range, `ncclAllGather` of the per-GPU partial sums, W-term addition on every device.

World size 1 exercises the same code path without the collective on any box; the 2-device cases need a box with at
least two GPUs and are skipped otherwise.  Every result is a group element and is compared bit for bit with the C oracle
or, at 2^20 points per GPU, with the known-discrete-log closed form.  Each test asserts the shape it claims before its
result: the window plan of every shard (`b200_multi_bases_plan`, the window restated from `msm_choose_plan`), the shard
ranges, and which windows hold digits (`msm_digits.py`).

What the layer adds to the single-context MSM and is pinned here: both entry points (`b200_multi_init` and the
per-rank `b200_multi_init_rank`), every window plan through the MSM's device-point epilogue (one point per shard left on
the device), `k_windows_to_point`'s Horner over split physical windows, `k_sum_partials` on cancelling and equal partials
and next to an empty shard, the context's own MSMs and replayed proofs around multi MSMs (each launch names its own
epilogue), the timing `bench.py` reads, and the refusals."""
import ast
import ctypes as C
import math
import os
import random
import threading

import numpy as np
import pytest
# torch before the first multi handle: the library binds libnccl.so.2 process-wide on its first NCCL call, and when that
# finds a system copy older than torch's, a later `import torch` fails on the NCCL symbols it needs.  Loaded first,
# torch's NCCL is the copy the library shares, as in bench.py and under torchrun.
import torch

import msm_digits as md
from renegade_b200 import _lib

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
R = md.R
SEED_BASES, SEED_SCALARS = 0xB200, 0x5CA1A8
PLAN_KEYS = ("window_bits", "digits", "physical_windows", "tables")


def _device_count():
    return torch.cuda.device_count()


def _need(world):
    if world > _device_count():
        pytest.skip(f"needs {world} GPUs")


def plan_of(m, mb, local=0) -> dict:
    """b200_multi_bases_plan of local device `local`'s shard."""
    arr = (C.c_int * 4)()
    _lib.check(m._lib.b200_multi_bases_plan(mb._h, local, arr))
    return dict(zip(PLAN_KEYS, arr))


def bench_multi_plan():
    """`multi_plan` as bench.py defines it, taken from its source without importing the script (whose import sets
    process-wide environment)."""
    with open(os.path.join(ROOT, "bench.py")) as f:
        tree = ast.parse(f.read())
    fn = next(n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name == "multi_plan")
    ns = {}
    exec(compile(ast.Module(body=[fn], type_ignores=[]), "bench.py", "exec"), ns)
    return ns["multi_plan"]


def assert_point(got, exp, what=""):
    (out, inf), (eout, einf) = got, exp
    assert inf == einf and (out == eout).all(), what


def identity():
    return np.zeros(8, dtype=np.uint64), True


def refused(code, fn, *args, **kw):
    with pytest.raises(_lib.B200Error) as ei:
        fn(*args, **kw)
    assert ei.value.code == code, ei.value
    return str(ei.value)


# ---- handles and inputs shared by the file ----------------------------------------------------------------------------
@pytest.fixture(scope="module")
def multi1():
    """single_process([0]): one process, one device, world 1."""
    from renegade_b200.sharded import MultiGpu
    m = MultiGpu.single_process([0])
    yield m
    m.close()


@pytest.fixture(scope="module")
def rank1():
    """for_rank(0, 0, 1, id): the one-process-per-GPU entry at world 1."""
    from renegade_b200.sharded import MultiGpu
    m = MultiGpu.for_rank(0, 0, 1, MultiGpu.unique_id())
    yield m
    m.close()


@pytest.fixture(scope="module")
def inputs(oracle):
    """n -> (known-discrete-log points, canonical scalars, Montgomery scalars, oracle MSM), made once per size."""
    cache = {}

    def get(n):
        if n not in cache:
            pts = oracle.known_dlog_bases(SEED_BASES, n)
            s = oracle.splitmix_fr(SEED_SCALARS, n, montgomery=False)
            cache[n] = (pts, s, oracle.splitmix_fr(SEED_SCALARS, n, montgomery=True), oracle.msm(pts, s))
        return cache[n]
    return get


@pytest.mark.parametrize("world", [1, 2])
def test_multi_msm_vs_oracle(oracle, world):
    _need(world)
    from renegade_b200.sharded import MultiGpu
    m = MultiGpu.single_process(list(range(world)))
    try:
        assert m.world == world and m.local_devices == world
        for n in (1, 5, 4099):           # n < world leaves a shard empty
            pts = oracle.known_dlog_bases(0xB200, n)
            s = oracle.splitmix_fr(0x5CA1A8, n, montgomery=False)
            mb = m.load_bases(pts, check_on_curve=True)
            assert len(mb) == n
            cuts = [mb.shard(i) for i in range(world)]
            assert cuts[0][0] == 0 and cuts[-1][1] == n
            out, inf = m.msm(mb, s)
            exp, einf = oracle.msm(pts, s)
            assert inf == einf and (out == exp).all(), (world, n)
            # Montgomery-form scalars (what `commit` is handed) and a zero vector (identity result)
            out, inf = m.msm(mb, oracle.splitmix_fr(0x5CA1A8, n, montgomery=True), montgomery=True)
            assert inf == einf and (out == exp).all()
            out, inf = m.msm(mb, np.zeros((n, 4), dtype=np.uint64))
            assert inf and not out.any()
            mb.free()
    finally:
        m.close()


# ---- 1 + 4. every plan through both entry points ----------------------------------------------------------------------
PLAN_SIZES = [1, 31, 4099, 110_000]  # 110 000 > 2^16: the throughput and latency models pick 17 and 16 there


def test_window_model_restatement_separates_the_plans():
    """The sizes above are where the plan's window tells the two automatic plans apart (n = 1 cannot)."""
    for n in PLAN_SIZES[1:]:
        assert md.choose_window(n, 0) != md.choose_window(n, 1), n
    assert [md.choose_window(n, 0) for n in (1, 31, 4099, 110_000)] == [8, 8, 13, 17]
    assert [md.choose_window(n, 1) for n in (1, 31, 4099, 110_000)] == [8, 10, 15, 16]


@pytest.mark.parametrize("entry", ["single_process", "for_rank"])
@pytest.mark.parametrize("source", ["load_bases", "known_dlog"])
@pytest.mark.parametrize("n", PLAN_SIZES)
@pytest.mark.parametrize("window_bits", [0, 1, 8, 12, 16, 23])
def test_multi_plans_match_oracle(request, ctx, inputs, entry, source, n, window_bits):
    """Every window plan with the window sums left on the device: the sharded MSM = oracle = the single-context MSM
    on bases loaded with the same window_bits, through both ways of making the handle."""
    m = request.getfixturevalue("multi1" if entry == "single_process" else "rank1")
    assert (m.world, m.local_devices, m.rank(0)) == (1, 1, 0)
    pts, s, s_mont, exp = inputs(n)
    mb = m.load_bases(pts, window_bits=window_bits) if source == "load_bases" else \
        m.known_dlog_bases(SEED_BASES, n, window_bits=window_bits)
    single = ctx.load_bases(pts, window_bits=window_bits)
    try:
        assert len(mb) == n and mb.shard(0) == (0, n)
        plan = plan_of(m, mb)
        assert plan == single.plan == md.expected_plan(n, window_bits), (plan, single.plan)
        assert_point(m.msm(mb, s), exp, "canonical")
        assert_point(m.msm(mb, s_mont, montgomery=True), exp, "montgomery")
        assert_point(ctx.msm(single, s), exp, "single context")
    finally:
        mb.free()
        single.free()


# ---- 2. physical windows: k_windows_to_point's device Horner --------------------------------------------------------
def scalars_in_phys_window(c, n_phys, p, count, rng):
    """Canonical scalars whose signed digits are all non-negative and lie in the windows w with w mod n_phys == p,
    every one of those windows non-zero (the top window's digit kept below r's top bits)."""
    W, half = md.num_windows(c), 1 << (c - 1)
    wins = [w for w in range(W) if w % n_phys == p]
    top_lim = R >> (c * (W - 1))
    out = []
    for _ in range(count):
        out.append(sum(rng.randint(1, min(half, top_lim - 1) if w == W - 1 else half) << (c * w) for w in wins))
    return out


def live_windows(vals, c):
    """Windows holding a non-zero digit in any of the scalars; asserts no carry leaves the top window."""
    live = set()
    for v in vals:
        digits, carry = md.signed_digits(v, c)
        assert carry == 0
        live |= {w for w, _, mag, _ in digits if mag}
    return live


def phys_scalar_sets(c, n_phys, n, rng):
    """(name, canonical scalars as ints) for the split-window tests, each with its window shape asserted."""
    W = md.num_windows(c)
    rand = [rng.randrange(R) for _ in range(n)]
    top = scalars_in_phys_window(c, n_phys, n_phys - 1, n, rng)
    low = scalars_in_phys_window(c, n_phys, 0, n, rng)
    assert {w % n_phys for w in live_windows(top, c)} == {n_phys - 1}
    assert {w % n_phys for w in live_windows(low, c)} == {0}
    assert len({w % n_phys for w in live_windows(rand, c)}) == n_phys  # random scalars reach every physical window
    assert live_windows(top, c) == {w for w in range(W) if w % n_phys == n_phys - 1}
    return [("random", rand), ("zero", [0] * n), ("top_phys_window_only", top), ("phys_window_0_only", low),
            ("r_minus_1", [R - 1] * n)]


@pytest.mark.parametrize("c", [8, 10])
@pytest.mark.parametrize("phys", ["2", "3", "W-1", "W"])
def test_multi_physical_windows(multi1, ctx, oracle, monkeypatch, c, phys):
    """B200_MSM_PHYS_WINDOWS (read per load) splits the tables: the multi path adds the physical windows' sums on the
    device (k_windows_to_point, c doublings per window, top window first), the single context on the host
    (msm_finish_batch).  Both must equal the oracle on scalars with digits in every, none, only the top and only the
    lowest physical window, r - 1, and one base with scalars 1 + 8 i (equal partial sums)."""
    W = md.num_windows(c)
    n_phys = {"2": 2, "3": 3, "W-1": W - 1, "W": W}[phys]
    monkeypatch.setenv("B200_MSM_PHYS_WINDOWS", str(n_phys))
    rng = random.Random(1000 * c + n_phys)
    n = 700
    pts = oracle.known_dlog_bases(0x51D0 + c, n)
    one = np.repeat(oracle.known_dlog_bases(0x0DE5, 1), n, axis=0)
    cases = [(pts, name, vals) for name, vals in phys_scalar_sets(c, n_phys, n, rng)]
    cases.append((one, "one_base_1_plus_8i", [1 + 8 * i for i in range(n)]))
    loaded = {}
    try:
        for key, p in (("pts", pts), ("one", one)):
            mb, single = multi1.load_bases(p, window_bits=c), ctx.load_bases(p, window_bits=c)
            loaded[key] = (mb, single)
            assert plan_of(multi1, mb) == single.plan == md.expected_plan(n, c, n_phys)
        for p, name, vals in cases:
            mb, single = loaded["pts" if p is pts else "one"]
            s = oracle.ints_to_array(vals)
            exp = oracle.msm(p, s)
            if name == "zero":
                assert exp[1]
            assert_point(multi1.msm(mb, s), exp, name)
            assert_point(ctx.msm(single, s), exp, name + " (single context)")
    finally:
        for mb, single in loaded.values():
            mb.free()
            single.free()


# ---- 3. the context around multi MSMs -------------------------------------------------------------------------------
TAU = 0x1c4e6a8b0d2f41638597a9cbedf0123456789abcdef0fedcba987654321
SEGMENTS = 7  # graph submissions per replayed proof


def _proof_setup(ctx, oracle, pyoracle, log_n):
    from renegade_b200 import synth
    from renegade_b200.backend import PlonkKzgSnark
    circ = synth.synth_circuit(log_n, num_inputs=5, seed=0x3171, check=True)
    srs = oracle.srs_from_tau(oracle.int_to_limbs(pyoracle.to_mont(TAU % pyoracle.R, pyoracle.R)), (1 << log_n) + 3)
    bases = ctx.load_bases(srs)
    pk = PlonkKzgSnark.preprocess(ctx, bases, log_n, circ.num_inputs, circ.selectors, circ.perm, circ.k)
    opk = oracle.plonk_preprocess(log_n, circ.selectors, circ.perm, circ.k, srs)
    return circ, srs, bases, pk, opk


def _proof_matches_oracle(ctx, oracle, log_n, setup, blind_seed):
    from renegade_b200 import synth
    from renegade_b200.backend import PlonkKzgSnark
    circ, srs, _, pk, opk = setup
    bl = synth.splitmix_blinders(blind_seed)
    proof, _ = PlonkKzgSnark.prove_with_link_hint(ctx, pk, circ.wires, circ.pub_inputs, bl)
    rc, oproof, _, _ = oracle.plonk_prove(log_n, circ.num_inputs, circ.k, opk, circ.wires, circ.pub_inputs, bl, srs)
    assert rc == 0 and bytes(proof) == bytes(oproof), blind_seed


def _batch_device(c, bases, d_scalars, n, stride, batch, montgomery):
    """b200_msm_batch_device through the context's own binding, as bench.py calls it."""
    out = np.zeros((batch, 8), dtype=np.uint64)
    inf = (C.c_int * batch)()
    _lib.check(c._lib.b200_msm_batch_device(c._h, bases._h, 0, C.c_void_p(d_scalars), n, stride, batch, int(montgomery),
                                            out.ctypes.data_as(C.c_void_p), inf))
    return [(out[i], bool(inf[i])) for i in range(batch)]


def test_context_msms_around_multi_msms(oracle, pyoracle):
    """multi_msm launches on the context's MSM scratch with the device-point epilogue, the context's own calls with theirs.
    On multi.ctx(0) of a fresh handle: first a proof whose graphs are captured BEFORE the context's first multi MSM and
    replayed after each of several (a replay must finish its commitments by the epilogue it captured, or it reads bit
    sums as window sums); then the context's MSMs on another base set (host and device scalars, batches through
    b200_msm_batch_device, canonical and Montgomery) interleaved with multi MSMs from host and device slices; then
    another proof.  Every result = oracle."""
    from renegade_b200.sharded import MultiGpu
    m = MultiGpu.single_process([0])
    mctx = m.ctx(0)
    setup, loaded = None, []
    try:
        # -- a replayed proof around multi MSMs: the multi MSM runs over the SRS points with the SRS's plan and device
        #    scalars, so it grows no scratch buffer the proof sized (a moved buffer would re-capture the graphs)
        log_n = 7
        setup = _proof_setup(mctx, oracle, pyoracle, log_n)
        srs = setup[1]
        ns = srs.shape[0]
        mb_srs = m.load_bases(srs)
        loaded.append(mb_srs)
        assert plan_of(m, mb_srs) == setup[2].plan
        s_srs = oracle.splitmix_fr(0x5125, ns, montgomery=False)
        exp_srs = oracle.msm(srs, s_srs)
        d_s_srs = torch.from_numpy(s_srs.view(np.int64)).to("cuda:0")
        torch.cuda.synchronize()
        mctx.use_graphs(True)
        _proof_matches_oracle(mctx, oracle, log_n, setup, 1)  # eager
        _proof_matches_oracle(mctx, oracle, log_n, setup, 2)  # captured and launched
        for i in range(3):
            assert_point(m.msm_local(mb_srs, [d_s_srs.data_ptr()], on_device=True), exp_srs, f"multi over the SRS {i}")
            g0 = mctx.graph_launches()
            _proof_matches_oracle(mctx, oracle, log_n, setup, 3 + i)  # replayed
            assert mctx.graph_launches() - g0 == SEGMENTS

        # -- the context's MSMs interleaved with multi MSMs
        n, nb = 4099, 3000
        pts = oracle.known_dlog_bases(SEED_BASES, n)
        s = oracle.splitmix_fr(SEED_SCALARS, n, montgomery=False)
        s_mont = oracle.splitmix_fr(SEED_SCALARS, n, montgomery=True)
        exp = oracle.msm(pts, s)
        other = oracle.known_dlog_bases(0xBEEF, nb)
        batch, stride = 3, nb + 8
        vecs = [oracle.splitmix_fr(0x7000 + i, nb, montgomery=False) for i in range(batch)]
        vexp = [oracle.msm(other, v) for v in vecs]
        packed = np.zeros((batch, stride, 4), dtype=np.uint64)
        packed_mont = np.zeros((batch, stride, 4), dtype=np.uint64)
        for i, v in enumerate(vecs):
            packed[i, :nb] = v
            packed_mont[i, :nb] = oracle.array_to_mont(oracle.FR, v)
        d_packed = torch.from_numpy(packed.view(np.int64)).to("cuda:0")
        d_packed_mont = torch.from_numpy(packed_mont.view(np.int64)).to("cuda:0")
        d_s = torch.from_numpy(s.view(np.int64)).to("cuda:0")
        d_s_mont = torch.from_numpy(s_mont.view(np.int64)).to("cuda:0")
        torch.cuda.synchronize()
        mb = m.load_bases(pts)
        loaded.append(mb)
        cb = mctx.load_bases(other)

        def multi_steps():
            yield "multi host canonical", lambda: m.msm(mb, s), exp
            yield "multi local host montgomery", lambda: m.msm_local(mb, [s_mont.ctypes.data], on_device=False, montgomery=True), exp
            yield "multi local device canonical", lambda: m.msm_local(mb, [d_s.data_ptr()], on_device=True), exp
            yield "multi local device montgomery", lambda: m.msm_local(mb, [d_s_mont.data_ptr()], on_device=True, montgomery=True), exp

        def ctx_steps():
            yield "ctx host", lambda: mctx.msm(cb, vecs[0]), vexp[0]
            yield "ctx device montgomery", lambda: mctx.msm_device(cb, d_packed_mont.data_ptr(), nb, montgomery=True), vexp[0]
            yield "ctx batch device", lambda: _batch_device(mctx, cb, d_packed.data_ptr(), nb, stride, batch, False), vexp
            yield "ctx batch device montgomery", lambda: _batch_device(mctx, cb, d_packed_mont.data_ptr(), nb, stride, batch, True), vexp

        try:
            order = [x for pair in zip(ctx_steps(), multi_steps()) for x in pair] + list(ctx_steps())
            for name, fn, want in order:
                got = fn()
                if isinstance(want, list):
                    for i, (g, w) in enumerate(zip(got, want)):
                        assert_point(g, w, f"{name} [{i}]")
                else:
                    assert_point(got, want, name)
            _proof_matches_oracle(mctx, oracle, log_n, setup, 10)
        finally:
            cb.free()
    finally:
        if setup is not None:
            setup[3].free()
            setup[2].free()
        for mb_ in loaded:
            mb_.free()
        m.close()


def test_context_and_multi_msms_from_two_threads(multi1, oracle):
    """One thread drives multi MSMs, another the context's own MSMs on multi.ctx(0), at once: every result exact,
    neither thread stuck (multi_msm holds the context's lock for its whole call)."""
    m, mctx = multi1, multi1.ctx(0)
    n, nb, rounds = 4099, 2500, 12
    pts = oracle.known_dlog_bases(SEED_BASES, n)
    s = oracle.splitmix_fr(SEED_SCALARS, n, montgomery=False)
    exp = oracle.msm(pts, s)
    other = oracle.known_dlog_bases(0xBEEF, nb)
    vecs = [oracle.splitmix_fr(0x7100 + i, nb, montgomery=False) for i in range(rounds)]
    vexp = [oracle.msm(other, v) for v in vecs]
    mb, cb = m.load_bases(pts), mctx.load_bases(other)
    results, errors = {"multi": [], "ctx": []}, []

    def run(name, fn):
        try:
            for i in range(rounds):
                results[name].append(fn(i))
        except Exception as e:  # surfaced below
            errors.append((name, e))

    threads = [threading.Thread(target=run, args=("multi", lambda i: m.msm(mb, s))),
               threading.Thread(target=run, args=("ctx", lambda i: mctx.msm(cb, vecs[i])))]
    try:
        for t in threads:
            t.start()
        for t in threads:
            t.join(timeout=300)
        assert not any(t.is_alive() for t in threads), "a thread did not finish"
        assert not errors, errors
        assert len(results["multi"]) == len(results["ctx"]) == rounds
        for got in results["multi"]:
            assert_point(got, exp, "multi")
        for i, got in enumerate(results["ctx"]):
            assert_point(got, vexp[i], f"ctx {i}")
    finally:
        cb.free()
        mb.free()


# ---- 5. the 2^20 leg bench.py times ---------------------------------------------------------------------------------
@pytest.mark.parametrize("world", [1, 2])
def test_multi_msm_2_20_per_gpu_closed_form(oracle, pyoracle, world):
    """world * 2^20 known-discrete-log bases generated on the devices: the sharded result must equal
    (sum a_i s_i mod r) * G.  With MSM timing on, as bench.py runs this leg, every device reports finite phases with
    the total at least each phase, one launch and 2^20 pairs per MSM; bench.py's `multi_plan` reads the plan the
    library reports."""
    _need(world)
    from renegade_b200.sharded import MultiGpu
    py = pyoracle
    per = 1 << 20
    n = world * per
    m = MultiGpu.single_process(list(range(world)))
    try:
        mb = m.known_dlog_bases(0xB200, n)
        assert bench_multi_plan()(m, mb) == plan_of(m, mb, 0) == md.expected_plan(per, 0)
        ctxs = [m.ctx(i) for i in range(world)]
        for c in ctxs:
            c.msm_timing(True)
            c.msm_timing_totals(reset=True)
        slices, keep = [], []
        for i in range(world):
            b, e = mb.shard(i)
            assert (b, e) == (i * per, (i + 1) * per)
            with torch.cuda.device(i):
                d = torch.empty((per, 4), dtype=torch.int64, device=f"cuda:{i}")
                torch.cuda.synchronize()
                m.ctx(i).splitmix_fr_device(0x5CA1A8, per, d.data_ptr(), montgomery=False, first=b)
            keep.append(d)
            slices.append(d.data_ptr())
        out, inf = m.msm_local(mb, slices, on_device=True)

        def check_timing(launches):
            for c in ctxs:
                ph = c.msm_timing(True)
                assert all(math.isfinite(v) and v >= 0 for v in ph.values()), ph
                assert ph["total"] > 0 and all(ph["total"] >= ph[k] for k in ("sort", "accumulate", "reduce")), ph
                t = c.msm_timing_totals()
                assert (t["launches"], t["pairs"]) == (launches, launches * per), t
                assert math.isfinite(t["accumulate_ms"]) and t["accumulate_ms"] > 0
        check_timing(1)
        a = oracle.array_to_ints(oracle.splitmix_fr(0xB200, n, False))
        s = oracle.array_to_ints(oracle.splitmix_fr(0x5CA1A8, n, False))
        k = sum(x * y for x, y in zip(a, s)) % py.R
        g = np.frombuffer(py.encode_g1_mont(py.G1_GEN), dtype=np.uint64)
        exp, _ = oracle.g1_mul(g, False, oracle.int_to_limbs(k))
        assert not inf and (out == exp).all()
        # host slices give the same point
        hs = [k_.cpu().numpy().view(np.uint64) for k_ in keep]
        out2, inf2 = m.msm_local(mb, [h.ctypes.data for h in hs], on_device=False)
        assert not inf2 and (out2 == exp).all()
        check_timing(2)
        for c in ctxs:
            c.msm_timing(False)
        mb.free()
    finally:
        m.close()


# ---- 6. partials that cancel, double, or sit next to an empty shard --------------------------------------------------
@pytest.fixture(params=[1, 2], ids=["world1", "world2"])
def multi_w(request):
    """single_process over `world` devices; world 1 computes the same sums in one shard, so the one-GPU box checks
    the expected values of the two-GPU cases."""
    _need(request.param)
    from renegade_b200.sharded import MultiGpu
    m = MultiGpu.single_process(list(range(request.param)))
    yield m
    m.close()


def test_multi_partials_cancel_and_double(multi_w, oracle):
    """Bases [P_0 … P_(m-1), P_0 … P_(m-1)]: at world 2 shard 0 holds the first copy and shard 1 the second.  Scalars
    [s, r - s] make the partials S and -S (k_sum_partials must return the identity), [s, s] make them equal (2S: the
    addition must take its doubling path)."""
    m, half = multi_w, 1500
    p = oracle.known_dlog_bases(0xCA7, half)
    pts = np.concatenate([p, p])
    s_int = oracle.array_to_ints(oracle.splitmix_fr(0x5EED, half, montgomery=False))
    s = oracle.ints_to_array(s_int)
    neg = oracle.ints_to_array([(R - v) % R for v in s_int])
    S, Sinf = oracle.msm(p, s)
    nS, nSinf = oracle.msm(p, neg)
    assert not Sinf and not nSinf and (nS[:4] == S[:4]).all() and not (nS[4:] == S[4:]).all()  # -S: same x, other y
    two_s = oracle.g1_add(S, False, S, False)
    mb = m.load_bases(pts)
    try:
        if m.world == 2:
            assert (mb.shard(0), mb.shard(1)) == ((0, half), (half, 2 * half))
        cancel, double = np.concatenate([s, neg]), np.concatenate([s, s])
        assert oracle.msm(pts, cancel)[1]
        assert_point(oracle.msm(pts, double), two_s)
        assert_point(m.msm(mb, cancel), identity(), "S + (-S)")
        assert_point(m.msm(mb, double), two_s, "S + S")
        assert_point(m.msm(mb, oracle.splitmix_fr(0x5EED, 2 * half, montgomery=False)),
                     oracle.msm(pts, oracle.splitmix_fr(0x5EED, 2 * half, montgomery=False)), "random")
    finally:
        mb.free()


def test_multi_one_point_next_to_an_empty_shard(multi_w, oracle):
    """n = 1: at world 2 shard 1 is empty (plan all zeros, no scalar slice needed) and contributes the identity
    record of msm_identity_point (k_windows_to_point(…, empty = 1))."""
    m = multi_w
    pts = oracle.known_dlog_bases(0x1, 1)
    mb = m.load_bases(pts, check_on_curve=True)
    try:
        cuts = [mb.shard(i) for i in range(m.world)]
        assert cuts == [(0, 1)] + [(1, 1)] * (m.world - 1)
        assert plan_of(m, mb, 0) == md.expected_plan(1, 0)
        for i in range(1, m.world):
            assert plan_of(m, mb, i) == dict.fromkeys(PLAN_KEYS, 0)
        for v in (1, 2, R - 1, 0xDEADBEEF, (R - 1) // 2):
            s = oracle.ints_to_array([v])
            exp = oracle.msm(pts, s)
            assert_point(m.msm(mb, s), exp, hex(v))
            assert_point(m.msm_local(mb, [s.ctypes.data] + [None] * (m.world - 1), on_device=False), exp, hex(v))
        assert_point(m.msm(mb, np.zeros((1, 4), dtype=np.uint64)), identity())
    finally:
        mb.free()


def test_multi_physical_windows_sharded(multi_w, oracle, monkeypatch):
    """Split physical windows (c = 10, 3 of them) on every shard: each device's Horner, then the W-term sum."""
    m, c, n_phys, n = multi_w, 10, 3, 3001
    monkeypatch.setenv("B200_MSM_PHYS_WINDOWS", str(n_phys))
    pts = oracle.known_dlog_bases(0xF00D, n)
    mb = m.load_bases(pts, window_bits=c)
    try:
        for i in range(m.world):
            b, e = mb.shard(i)
            assert plan_of(m, mb, i) == md.expected_plan(e - b, c, n_phys)
        rng = random.Random(77)
        for name, vals in phys_scalar_sets(c, n_phys, n, rng):
            s = oracle.ints_to_array(vals)
            assert_point(m.msm(mb, s), oracle.msm(pts, s), name)
    finally:
        mb.free()


# ---- 7. refusals ----------------------------------------------------------------------------------------------------
def test_multi_refusals_leave_the_handle_usable(multi1, oracle):
    """Each refusal returns its documented code before any work, and the handle runs a correct MSM after it."""
    from renegade_b200.sharded import MultiGpu
    m, n = multi1, 257
    INVALID, NOT_ON_CURVE = _lib.B200_ERR_INVALID, _lib.B200_ERR_NOT_ON_CURVE
    pts = oracle.known_dlog_bases(SEED_BASES, n)
    s = oracle.splitmix_fr(SEED_SCALARS, n, montgomery=False)
    exp = oracle.msm(pts, s)
    mb = m.load_bases(pts)
    lib = m._lib

    def still_works():
        assert_point(m.msm(mb, s), exp, "after a refusal")

    try:
        # scalar count other than the loaded bases
        for k in (n - 1, n + 1, 0):
            msg = refused(INVALID, m.msm, mb, oracle.splitmix_fr(SEED_SCALARS, k, montgomery=False))
            assert "differs from the loaded bases" in msg
            still_works()
        # a NULL slice for a non-empty shard, host or device
        for on_device in (False, True):
            refused(INVALID, m.msm_local, mb, [None], on_device=on_device)
            still_works()
        # no points; windows outside 0, 1, 8 … 23
        refused(INVALID, m.load_bases, np.zeros((0, 8), dtype=np.uint64))
        still_works()
        refused(INVALID, m.known_dlog_bases, SEED_BASES, 0)
        still_works()
        for wb in (2, 7, 24, -1):
            refused(INVALID, m.load_bases, pts, window_bits=wb)
            refused(INVALID, m.known_dlog_bases, SEED_BASES, n, window_bits=wb)
            still_works()
        # a point off the curve under check_on_curve; without the check the same points load
        bad = pts.copy()
        bad[n // 2, 0] ^= np.uint64(1)
        assert not oracle.g1_on_curve(bad[n // 2])
        assert "not on curve" in refused(NOT_ON_CURVE, m.load_bases, bad, check_on_curve=True)
        still_works()
        fresh = m.load_bases(pts, check_on_curve=True)
        assert_point(m.msm(fresh, s), exp, "fresh bases after the off-curve refusal")
        fresh.free()
        # handles: 0 or 65 devices; per-rank: bad rank, bad world, NULL id
        refused(INVALID, MultiGpu.single_process, [])
        refused(INVALID, MultiGpu.single_process, [0] * 65)
        uid = MultiGpu.unique_id()
        for dev, rank, world in ((0, 1, 1), (0, -1, 1), (0, 0, 0), (0, 0, -2), (0, 2, 2)):
            refused(INVALID, MultiGpu.for_rank, dev, rank, world, uid)
        h = C.c_void_p()
        assert lib.b200_multi_init_rank(0, 0, 1, None, C.byref(h)) == INVALID and not h.value
        # the accessors on NULL handles and out-of-range local indices
        assert (lib.b200_multi_world(None), lib.b200_multi_local_devices(None), lib.b200_multi_rank(None, 0)) == (0, 0, -1)
        assert lib.b200_multi_rank(m._h, 1) == -1 and not lib.b200_multi_ctx(m._h, 1)
        arr = (C.c_int * 4)()
        assert lib.b200_multi_bases_plan(mb._h, 1, arr) == INVALID and lib.b200_multi_bases_plan(None, 0, arr) == INVALID
        still_works()
    finally:
        mb.free()


def test_nccl_is_bound_at_run_time():
    v = C.c_int(0)
    _lib.check(_lib.load().b200_nccl_version(C.byref(v)))
    assert v.value >= 22000
