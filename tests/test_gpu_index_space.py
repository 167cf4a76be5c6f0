"""GPU: the MSM and the NTT at the top of the sizes their C ABI accepts, where integer kernels go wrong: 2^26 bases (the
point index fills all 26 bits of a bucket entry), window tables split by the memory budget, bucket-entry offsets past
2^31 and up to just below 2^32, the three launch guards of msm_launch_batch, domains of 2^23 … 2^28 (2^28 is the only
size that uses the two-adic root unsquared), and NTT batches past CUDA's 65 535 grid rows.

Expected values never come from the library: MSMs over known-dlog bases a_i G with SplitMix scalars s_i equal
(sum a_i s_i mod r) G, the sum by the C oracle's orc_fr_dot and the point by orc_g1_mul; NTTs are compared with orc_ntt
or, at 2^27 and 2^28, with sums of a few powers of the root computed with Python integers.

Every test runs on a context of its own, closed at its end (a context keeps its NTT domains for its life: 24 GiB at
2^28), and skips with the numbers when the GPU has less free memory than the test needs."""
import contextlib
import ctypes as C
import gc
import os
import random
import re
import time

import numpy as np
import pytest
import torch

import msm_digits as md
import renegade_b200 as rb
from renegade_b200 import _lib

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
R = md.R
MONT = (1 << 256) % R
MONT_INV = pow(MONT, -1, R)
GiB = 1 << 30
SEED_BASES, SEED_SCALARS, SEED_NTT = 0xB200, 0x5CA1A8, 0x1177
MAX_BASES = 1 << md.IDX_BITS


def _source(name: str) -> str:
    with open(os.path.join(ROOT, "renegade_b200", "csrc", name)) as f:
        return f.read()


@contextlib.contextmanager
def dedicated_context(need_bytes: int, what: str):
    """A fresh context for one large test, closed (with its domains and scratch) and torch's cache emptied after it.
    Tensors of an earlier test can outlive it in a reference cycle (a caught exception's traceback holds the test's
    frame): collected first, so that the free memory seen here is what this test can use."""
    gc.collect()
    torch.cuda.empty_cache()
    free, total = torch.cuda.mem_get_info()
    if free < need_bytes:
        pytest.skip(f"{what} wants {need_bytes >> 20} MiB free, the GPU has {free >> 20} of {total >> 20} MiB free")
    print(f"{what}: {free >> 20} of {total >> 20} MiB free, {need_bytes >> 20} MiB wanted")
    ctx = rb.Context(0)
    try:
        yield ctx
    finally:
        ctx.close()
        torch.cuda.synchronize()
        torch.cuda.empty_cache()


def refused(fn, *args, **kw):
    with pytest.raises(_lib.B200Error) as ei:
        fn(*args, **kw)
    assert ei.value.code == _lib.B200_ERR_INVALID, ei.value


def closed_form(oracle, pyoracle, n: int, first_a: int = 0, first_s: int = 0):
    """sum_{i < n} s_{first_s + i} P_{first_a + i} for P_i = a_i G: (sum a_i s_i mod r) G, and whether it is the
    identity."""
    k = oracle.fr_dot(SEED_BASES, SEED_SCALARS, n, first_a, first_s)
    g = np.frombuffer(pyoracle.encode_g1_mont(pyoracle.G1_GEN), dtype=np.uint64)
    return oracle.g1_mul(g, False, oracle.int_to_limbs(k))


def assert_point(got, exp, what=""):
    (out, inf), (eout, einf) = got, exp
    assert inf == einf and (np.asarray(out) == eout).all(), what


def rows_u64(t: torch.Tensor) -> np.ndarray:
    return t.cpu().numpy().view(np.uint64)


def msm_batch(ctx, bases, d_scalars: int, n: int, stride: int, batch: int, base_off: int = 0):
    out = np.zeros((batch, 8), dtype=np.uint64)
    inf = (C.c_int * batch)()
    _lib.check(ctx._lib.b200_msm_batch_device(ctx._h, bases._h, base_off, C.c_void_p(d_scalars), n, stride, batch, 0,
                                              out.ctypes.data_as(C.c_void_p), inf))
    return [(out[i], bool(inf[i])) for i in range(batch)]


# ---- 1. MSM over 2^26 bases ------------------------------------------------------------------------------------------
def test_msm_2_26_bases(oracle, pyoracle, monkeypatch):
    """2^26 known-dlog bases generated on the device (sampled against the oracle at 0, 2^24, 2^25 - 1, 2^25 and the
    last), loaded at exactly the limit, 2^26 + 1 refused by both loaders; the MSM of 2^26 SplitMix scalars under the
    automatic plan (tables split by the memory budget) and under a forced split equals the closed form, and so does
    the MSM of the last five bases, whose point indices fill all 26 bits of a bucket entry."""
    n = MAX_BASES
    c = md.choose_window(n, 0)
    W = md.num_windows(c)
    idx = md.index_space(n, c, 1, 1)
    # points and scalars, one table, the MSM scratch (entries, segment sums and their order, buckets), 2 GiB of slack
    need = n * 64 + n * 32 + n * 64 + idx["entries"] * 4 + idx["segments"] * 136 + (W << (c - 1)) * 160 + 2 * GiB
    with dedicated_context(need, "MSM of 2^26 points") as ctx:
        t0 = time.time()
        d_pts = torch.empty((n, 8), dtype=torch.int64, device="cuda")
        d_s = torch.empty((n, 4), dtype=torch.int64, device="cuda")
        torch.cuda.synchronize()
        ctx.known_dlog_bases_device(SEED_BASES, n, d_pts.data_ptr())
        ctx.splitmix_fr_device(SEED_SCALARS, n, d_s.data_ptr(), montgomery=False)
        for i in (0, 1 << 24, (1 << 25) - 1, 1 << 25, n - 1):
            assert (rows_u64(d_pts[i:i + 1]) == oracle.known_dlog_bases(SEED_BASES, 1, first=i)).all(), i
            assert (rows_u64(d_s[i:i + 1]) == oracle.splitmix_fr(SEED_SCALARS, 1, False, first=i)).all(), i
        # one point past the limit: refused by the device and the host loader before they read or allocate anything
        refused(ctx.load_bases_device, d_pts.data_ptr(), n + 1)
        refused(ctx.load_bases, np.empty((n + 1, 8), dtype=np.uint64))
        exp = closed_form(oracle, pyoracle, n)
        exp_top = closed_form(oracle, pyoracle, 5, n - 5, n - 5)
        free_at_load = torch.cuda.mem_get_info()[0]
        bases = ctx.load_bases_device(d_pts.data_ptr(), n)
        plan = bases.plan
        print(f"2^26 points, {free_at_load >> 20} MiB free at load: plan {plan}")
        assert plan == md.expected_plan(n, 0, plan["physical_windows"])
        assert plan["tables"] * n * 64 <= free_at_load // 2 or plan["physical_windows"] == W
        assert_point(ctx.msm_device(bases, d_s.data_ptr(), n), exp, "2^26 points, automatic plan")
        assert_point(ctx.msm_device(bases, d_s.data_ptr() + 32 * (n - 5), 5, base_off=n - 5), exp_top, "top five")
        bases.free()
        # a forced split into two tables (c = 20: 7 of the 13 windows physical), or into one where the budget chose two
        forced = (W + 1) // 2 if plan["physical_windows"] != (W + 1) // 2 else W
        monkeypatch.setenv("B200_MSM_PHYS_WINDOWS", str(forced))
        bases = ctx.load_bases_device(d_pts.data_ptr(), n)
        split = bases.plan
        print(f"2^26 points, B200_MSM_PHYS_WINDOWS={forced}: plan {split}")
        assert split["physical_windows"] >= forced and split != plan
        assert_point(ctx.msm_device(bases, d_s.data_ptr(), n), exp, f"2^26 points, split {split}")
        top = ctx.msm_device(bases, d_s.data_ptr() + 32 * (n - 5), 5, base_off=n - 5)
        assert_point(top, exp_top, "top five, split")
        bases.free()
        print(f"2^26-point MSM checks: {time.time() - t0:.1f} s")


# ---- 2. MSM offsets past 2^31 and the launch guards ------------------------------------------------------------------
@pytest.mark.parametrize("batch", [40, 63])
def test_msm_entry_offsets_past_2_31(oracle, pyoracle, batch):
    """A batch of MSMs of 2^22 points at c = 16 whose bucket entries number past 2^31 (40 MSMs) and just below 2^32
    (63): every offset, cursor and segment bound of the pipeline holds bit 31 for the later buckets.  Every member equals
    its closed form."""
    n, c = 1 << 22, 16
    idx = md.index_space(n, c, 1, batch)
    assert idx["entries"] > (1 << 31) and not idx["refused"], idx
    need = (md.num_windows(c) * n * 64 + n * 64 + batch * n * 32 + idx["entries"] * 4 + idx["segments"] * 136
            + idx["buckets"] * 160 + 2 * GiB)
    with dedicated_context(need, f"{batch} MSMs of 2^22 points") as ctx:
        t0 = time.time()
        d_pts = torch.empty((n, 8), dtype=torch.int64, device="cuda")
        torch.cuda.synchronize()
        ctx.known_dlog_bases_device(SEED_BASES, n, d_pts.data_ptr())
        bases = ctx.load_bases_device(d_pts.data_ptr(), n, window_bits=c)
        del d_pts
        torch.cuda.empty_cache()
        assert bases.plan == md.expected_plan(n, c, 1)
        d_s = torch.empty((batch * n, 4), dtype=torch.int64, device="cuda")
        torch.cuda.synchronize()
        ctx.splitmix_fr_device(SEED_SCALARS, batch * n, d_s.data_ptr(), montgomery=False)
        got = msm_batch(ctx, bases, d_s.data_ptr(), n, n, batch)
        t_gpu = time.time() - t0
        for k in range(batch):
            assert_point(got[k], closed_form(oracle, pyoracle, n, 0, k * n), f"member {k} of {batch}")
        bases.free()
        print(f"{batch} x 2^22 ({idx['entries']} worst-case entries): {t_gpu:.1f} s on the GPU, "
              f"{time.time() - t0 - t_gpu:.1f} s of closed forms")


def test_msm_launch_guards(oracle, pyoracle, monkeypatch):
    """One shape per guard of msm_launch_batch (msm_digits.GUARD_SHAPES: worst-case entries exactly 2^32, buckets past
    2^31, segments past 2^30 with the other two inside), each refused with B200_ERR_INVALID, and a correct batch MSM on
    the same context after each refusal."""
    n_e, c_e, phys_e, batch_e = md.GUARD_SHAPES["entries"]
    need = n_e * 64 * 2 + batch_e * n_e * 32 + GiB
    with dedicated_context(need, "MSM launch guards") as ctx:
        d_pts = torch.empty((n_e, 8), dtype=torch.int64, device="cuda")
        torch.cuda.synchronize()
        ctx.known_dlog_bases_device(SEED_BASES, n_e, d_pts.data_ptr())
        monkeypatch.setenv("B200_MSM_PHYS_WINDOWS", str(phys_e))
        big = ctx.load_bases_device(d_pts.data_ptr(), n_e, window_bits=c_e)
        assert big.plan == md.expected_plan(n_e, c_e, phys_e)
        del d_pts
        # valid scalars for every member, so that a guard that let the launch through would compute, not fault
        d_zero = torch.zeros((batch_e * n_e, 4), dtype=torch.int64, device="cuda")
        small_n, small_batch = 4096, 2
        d_s = torch.empty((small_batch * small_n, 4), dtype=torch.int64, device="cuda")
        torch.cuda.synchronize()
        ctx.splitmix_fr_device(SEED_SCALARS, small_batch * small_n, d_s.data_ptr(), montgomery=False)
        exp = [closed_form(oracle, pyoracle, small_n, 0, k * small_n) for k in range(small_batch)]

        def still_correct(what):
            got = msm_batch(ctx, big, d_s.data_ptr(), small_n, small_n, small_batch)
            for k in range(small_batch):
                assert_point(got[k], exp[k], f"after the {what} refusal, member {k}")

        assert md.index_space(n_e, c_e, phys_e, batch_e)["entries"] == 1 << 32
        refused(msm_batch, ctx, big, d_zero.data_ptr(), n_e, n_e, batch_e)
        still_correct("entries")
        monkeypatch.setenv("B200_MSM_PHYS_WINDOWS", "12")
        one = ctx.load_bases(oracle.known_dlog_bases(SEED_BASES, 1), window_bits=23)
        for name in ("buckets", "segments"):
            n, c, phys, batch = md.GUARD_SHAPES[name]
            assert one.plan == md.expected_plan(n, c, phys)
            idx = md.index_space(n, c, phys, batch)
            assert idx["refused"] and idx["entries"] < 1 << 32, idx
            refused(msm_batch, ctx, one, d_zero.data_ptr(), n, n, batch)
            still_correct(name)
        one.free()
        big.free()


# ---- 3. NTT at 2^23 … 2^28 -------------------------------------------------------------------------------------------
VARIANTS = [(False, False), (True, False), (False, True), (True, True)]  # (inverse, coset)


def ntt_need(log_n: int, copies: int) -> int:
    """data copies, the scratch, the domain's twiddles (n / 2 per direction) and coset tables (n per direction)"""
    return ((copies + 1) * 32 + 32 + 64) << log_n


@pytest.mark.parametrize("log_n", [23, 24, 25])
def test_ntt_random_vs_oracle(oracle, log_n):
    """Random inputs, all four variants, bit for bit against orc_ntt, at three passes of 8 / 8 / 7, 8 / 8 / 8 and
    9 / 8 / 8 stages."""
    n = 1 << log_n
    with dedicated_context(ntt_need(log_n, 1) + GiB, f"NTT 2^{log_n}") as ctx:
        x = oracle.splitmix_fr(SEED_NTT + log_n, n, montgomery=True)
        d = torch.empty((n, 4), dtype=torch.int64, device="cuda")
        t_gpu = t_orc = 0.0
        for inverse, coset in VARIANTS:
            d.copy_(torch.from_numpy(x.view(np.int64)))
            torch.cuda.synchronize()
            t0 = time.time()
            ctx.ntt_device(d.data_ptr(), log_n, inverse, coset)
            t1 = time.time()
            exp = oracle.ntt(x, inverse, coset)
            t_orc += time.time() - t1
            t_gpu += t1 - t0
            assert (rows_u64(d) == exp).all(), (log_n, inverse, coset)
        print(f"NTT 2^{log_n}: four variants, {t_gpu:.2f} s on the GPU, {t_orc:.1f} s in the oracle")


def sparse_positions(n: int) -> list[int]:
    """16 input positions across the tile (2^10) and pass edges: the first pass of 2^27 / 2^28 spans 9 / 10 stages"""
    return sorted({0, 1, (1 << 9) - 1, (1 << 9) + 1, (1 << 10) - 1, 1 << 10, (1 << 10) + 1, 1 << 19, (1 << 19) + 1,
                   (1 << 20) - 1, 1 << 20, (1 << 20) + 1, n // 2, n // 2 + 1, n - 2, n - 1})


def sample_outputs(n: int, rng: random.Random, count: int = 4096) -> list[int]:
    edges = {0, 1, n // 2, n - 1}
    for k in range(1, n.bit_length() - 1):
        edges |= {(1 << k) - 1, 1 << k, (1 << k) + 1, n - (1 << k)}
    out = sorted(edges)
    return sorted(set(out) | set(rng.randrange(n) for _ in range(count - len(out))))


def sparse_expected(vals: dict, j: int, n: int, inverse: bool, coset: bool) -> int:
    """Output j of the transform of the sparse vector {position: value}, canonical, from the definitions: forward
    sum x_t w^(p_t j), coset forward sum x_t 5^p_t w^(p_t j), inverse n^-1 sum x_t w^(-p_t j), coset inverse the
    inverse times 5^-j; w = 5^((r - 1) / n)."""
    w = pow(5, (R - 1) // n, R)
    if inverse:
        w = pow(w, -1, R)
    acc = 0
    for p, x in vals.items():
        if coset and not inverse:
            x = x * pow(5, p, R)
        acc += x * pow(w, (p * j) % n, R)
    acc %= R
    if inverse:
        acc = acc * pow(n, -1, R) % R
        if coset:
            acc = acc * pow(5, -j, R) % R
    return acc


def oracle_limbs(v: int) -> np.ndarray:
    return np.array([(v >> (64 * i)) & 0xFFFFFFFFFFFFFFFF for i in range(4)], dtype=np.uint64)


def to_int(limbs) -> int:
    return sum(int(v) << (64 * i) for i, v in enumerate(np.asarray(limbs, dtype=np.uint64)))


@pytest.mark.parametrize("log_n", [27, 28])
def test_ntt_sparse_and_round_trips(log_n):
    """At 2^27 and 2^28 (three passes of 9 / 9 / 9 and 10 / 9 / 9 stages; 2^28 uses the two-adic root itself): the
    domain's generator has order exactly n; a vector of 16 non-zeros at tile and pass edges, through all four variants,
    matches the definition at ~4096 sampled outputs (0, 1, n/2, n - 1 and every power of two and its neighbours among
    them); and random vectors come back bit for bit through iNTT(NTT(x)) and coset-iNTT(coset-NTT(x))."""
    n = 1 << log_n
    rng = random.Random(log_n)
    with dedicated_context(ntt_need(log_n, 2) + GiB, f"NTT 2^{log_n}") as ctx:
        t0 = time.time()
        g = to_int(ctx.domain_generator(log_n)) * MONT_INV % R
        assert pow(g, n >> 1, R) == R - 1 and pow(g, n, R) == 1, "generator of order other than n"
        assert g == pow(5, (R - 1) >> log_n, R)
        vals = {p: rng.randrange(1, R) for p in sparse_positions(n)}
        js = sample_outputs(n, rng)
        d = torch.empty((n, 4), dtype=torch.int64, device="cuda")
        pos = torch.tensor(list(vals), dtype=torch.int64, device="cuda")
        src = torch.from_numpy(np.stack([oracle_limbs(v * MONT % R) for v in vals.values()]).view(np.int64)).cuda()
        jt = torch.tensor(js, dtype=torch.int64, device="cuda")
        for inverse, coset in VARIANTS:
            d.zero_()
            d[pos] = src
            torch.cuda.synchronize()
            ctx.ntt_device(d.data_ptr(), log_n, inverse, coset)
            got = rows_u64(d[jt])
            for j, row in zip(js, got):
                exp = sparse_expected(vals, j, n, inverse, coset)
                assert to_int(row) * MONT_INV % R == exp, (log_n, inverse, coset, j)
        # round trips on random device vectors
        x = torch.empty((n, 4), dtype=torch.int64, device="cuda")
        torch.cuda.synchronize()
        ctx.splitmix_fr_device(SEED_NTT + log_n, n, x.data_ptr(), montgomery=True)
        for coset in (False, True):
            d.copy_(x)
            torch.cuda.synchronize()
            ctx.ntt_device(d.data_ptr(), log_n, False, coset)
            assert not torch.equal(d, x)
            ctx.ntt_device(d.data_ptr(), log_n, True, coset)
            assert torch.equal(d, x), ("round trip", log_n, coset)
        print(f"NTT 2^{log_n}: sparse and round-trip checks in {time.time() - t0:.1f} s")


# ---- 4. NTT batches past 65 535 --------------------------------------------------------------------------------------
def test_grid_y_bounds_in_the_sources():
    """Every launch that puts a batch on gridDim.y (capped at 65 535 by CUDA) bounds it: the NTT launches at most
    kMaxBatchPerLaunch = 65 535 transforms per grid, b200_msm_batch_device takes at most 64 MSMs (gridDim.y of the digit
    kernels, and 32 physical windows times 64 in the bit sums), the prover and link batches run in chunks of at most
    kMaxBatchChunk = 64."""
    ntt = _source("ntt.cu")
    assert re.search(r"constexpr unsigned kMaxBatchPerLaunch = 65535;", ntt)
    assert re.search(r"first \+= kMaxBatchPerLaunch", ntt)
    assert re.search(r"dim3 grid\(\(unsigned\)\(\(\(size_t\)1 << L\) >> e_log\), batch\);", ntt)
    assert re.search(r"batch > 64 \|\| stride < n\) return B200_ERR_INVALID;", _source("api.cu"))
    assert re.search(r"constexpr size_t kMaxBatchChunk = 64;", _source("plonk.cu"))


NTT_BATCHES = [(log_n, batch) for log_n in (1, 2, 10) for batch in (65535, 65536, 65537, 1 << 17)] + [(11, 65537)]
PERIOD = 97  # distinct rows; prime, so no chunk of 65 535 rows lines up with the pattern


@pytest.mark.parametrize("log_n, batch", NTT_BATCHES)
def test_ntt_batches_past_grid_rows(oracle, log_n, batch):
    """b200_ntt_device on batches around and past 65 535 transforms, stride n + 5: every row equals orc_ntt of its input
    (row r holds input r mod 97), all four variants, and the five padding elements after each row stay untouched."""
    n, stride = 1 << log_n, (1 << log_n) + 5
    total = batch * stride * 32
    need = total * (3 if log_n > 10 else 2) + ntt_need(log_n, 0) + GiB
    with dedicated_context(need, f"NTT batch {batch} x 2^{log_n}") as ctx:
        x = oracle.splitmix_fr(SEED_NTT + batch, PERIOD * n, montgomery=True).reshape(PERIOD, n, 4)
        rows = torch.arange(batch, device="cuda") % PERIOD
        src = torch.from_numpy(x.view(np.int64)).cuda()
        pad = torch.full((batch, stride - n, 4), 0x5A5A5A5A5A5A5A5A, dtype=torch.int64, device="cuda")
        d = torch.empty((batch, stride, 4), dtype=torch.int64, device="cuda")
        for inverse, coset in VARIANTS:
            exp = np.stack([oracle.ntt(x[p], inverse, coset) for p in range(PERIOD)])
            exp = torch.from_numpy(exp.view(np.int64)).cuda()
            d[:, :n] = src[rows]
            d[:, n:] = pad
            torch.cuda.synchronize()
            ctx.ntt_device(d.data_ptr(), log_n, inverse, coset, batch=batch, stride=stride)
            torch.cuda.synchronize()
            assert torch.equal(d[:, n:], pad), ("padding", inverse, coset)
            bad = (d[:, :n] != exp[rows]).reshape(batch, -1).any(dim=1).nonzero().flatten()
            assert bad.numel() == 0, (inverse, coset, bad[:8].tolist(), bad.numel())
