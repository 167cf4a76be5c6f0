"""GPU parity: NTT / iNTT / coset variants through the C ABI vs the oracle (bit-exact) at every size up to 2^22 —
one, two and three passes — the golden known answers, size-independent properties, twiddle-sensitive transforms of
unit vectors at 2^22 and 2^24 against Python `pow`, structured inputs, and batches whose padding must stay untouched."""
import os
import random
import re

import numpy as np
import pytest

import renegade_b200 as rb

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
R = 0x30644E72E131A029B85045B68181585D2833E84879B97091_43E1F593F0000001
MONT = 1 << 256
VARIANTS = [(False, False), (False, True), (True, False), (True, True)]  # (inverse, coset)


def H(s):
    return int(s, 16)


def passes(log_n: int) -> int:
    """Passes of ntt_device: ceil(log n / kTileLog), the tile size read from ntt.cu."""
    with open(os.path.join(ROOT, "renegade_b200", "csrc", "ntt.cu")) as f:
        tile_log = int(re.search(r"#define B200_NTT_TILE_LOG (\d+)", f.read()).group(1))
    return -(-log_n // tile_log)


def limbs(v: int) -> list[int]:
    return [(v >> (64 * k)) & ((1 << 64) - 1) for k in range(4)]


def to_int(row) -> int:
    return sum(int(x) << (64 * k) for k, x in enumerate(np.asarray(row, dtype=np.uint64).reshape(4)))


@pytest.mark.parametrize("log_n", range(23))
def test_ntt_matches_oracle(ctx, oracle, log_n):
    n = 1 << log_n
    if log_n >= 21:
        assert passes(log_n) == 3  # a middle pass whose tile has lo > 0 and hi < log n
    x = oracle.splitmix_fr(0x1177, n, montgomery=True)
    for inverse, coset in VARIANTS:
        got = ctx.ntt(x, inverse=inverse, coset=coset)
        exp = oracle.ntt(x, inverse=inverse, coset=coset)
        assert (got == exp).all(), (log_n, inverse, coset)


@pytest.mark.parametrize("log_n", [22, 24])
def test_ntt_unit_vectors_against_pow(ctx, oracle, log_n):
    """NTT(delta_k)[j] = w^(jk), coset: 5^k w^(jk), inverse: n^-1 w^(-jk), coset inverse: n^-1 5^-j w^(-jk), for
    k = 1, n/2 - 1, n - 1 at sampled j.  delta_0 and constant inputs multiply every twiddle by zero; these do not, so a
    transform on another root of unity (a twiddle stride off in both directions, a pass on the wrong table) fails."""
    import torch
    n = 1 << log_n
    assert passes(log_n) == 3
    w_mont = ctx.domain_generator(log_n)
    assert (w_mont == oracle.domain_generator(log_n)).all()
    w = to_int(w_mont) * pow(MONT, -1, R) % R
    assert pow(w, n, R) == 1 and pow(w, n // 2, R) == R - 1  # a primitive n-th root of unity
    n_inv, g = pow(n, -1, R), 5
    rng = random.Random(log_n)
    js = sorted({0, 1, 2, n // 2 - 1, n // 2, n // 2 + 1, n - 1} | {rng.randrange(n) for _ in range(9)})
    idx = torch.tensor(js, device="cuda")
    one = torch.from_numpy(np.array(limbs(MONT % R), dtype=np.uint64).view(np.int64)).cuda()
    d = torch.empty((n, 4), dtype=torch.int64, device="cuda")
    for k in (1, n // 2 - 1, n - 1):
        for inverse, coset in VARIANTS:
            d.zero_()
            d[k] = one
            torch.cuda.synchronize()
            ctx.ntt_device(d.data_ptr(), log_n, inverse=inverse, coset=coset)
            got = d[idx].cpu().numpy().view(np.uint64)
            for row, j in zip(got, js):
                if not inverse:
                    v = pow(w, j * k, R) * (pow(g, k, R) if coset else 1)
                else:
                    v = n_inv * pow(w, -j * k, R) * (pow(g, -j, R) if coset else 1)
                assert to_int(row) == v * MONT % R, (log_n, k, inverse, coset, j)


@pytest.mark.parametrize("log_n", [16, 21])
def test_ntt_structured_inputs(ctx, oracle, log_n):
    """All r - 1 (the largest residue in every lane) and alternating 0 / r - 1, at a two- and a three-pass size."""
    n = 1 << log_n
    assert passes(log_n) == (2 if log_n <= 20 else 3)
    top = np.array(limbs(R - 1), dtype=np.uint64)
    full = np.tile(top, (n, 1))
    alt = full.copy()
    alt[0::2] = 0
    for x in (full, alt):
        for inverse, coset in VARIANTS:
            got = ctx.ntt(x, inverse=inverse, coset=coset)
            assert (got == oracle.ntt(x, inverse=inverse, coset=coset)).all(), (log_n, inverse, coset)


def test_ntt_golden(ctx, oracle, pyoracle, kat):
    py = pyoracle
    for rec in kat["ntt"]:
        xm = oracle.ints_to_array([py.to_mont(H(v), py.R) for v in rec["x"]])
        dom = rb.Radix2EvaluationDomain(ctx, len(rec["x"]))
        for key, fn in (("fft", dom.fft), ("ifft", dom.ifft), ("coset_fft", dom.coset_fft)):
            got = [py.from_mont(v, py.R) for v in oracle.array_to_ints(fn(xm))]
            assert got == [H(v) for v in rec[key]], (rec["log_n"], key)


def test_domain_matches_reference_shape(ctx, oracle):
    dom = rb.Radix2EvaluationDomain(ctx, (1 << 16) + 3)  # ark-poly rounds up to the next power of 2
    assert dom.size == 1 << 17 and dom.log_size_of_group == 17
    assert (dom.group_gen == oracle.domain_generator(17)).all()
    # fewer coefficients than the domain: zero-padded like ark-poly
    x = oracle.splitmix_fr(0x77, 100, montgomery=True)
    d2 = rb.Radix2EvaluationDomain(ctx, 100)
    padded = np.concatenate([x, np.zeros((28, 4), dtype=np.uint64)])
    assert (d2.fft(x) == oracle.ntt(padded)).all()


def test_ntt_2_20_full_size(ctx, oracle):
    """BASELINE.json config 3: 2^20 NTT + iNTT round trip, plus exact oracle equality
    (the C oracle does 2^20 in well under a second)."""
    n = 1 << 20
    x = oracle.splitmix_fr(0x1177, n, montgomery=True)
    y = ctx.ntt(x)
    assert (y == oracle.ntt(x)).all()
    assert (ctx.ntt(y, inverse=True) == x).all()
    yc = ctx.ntt(x, coset=True)
    assert (ctx.ntt(yc, inverse=True, coset=True) == x).all()


def test_ntt_properties_2_22(ctx, oracle, pyoracle):
    """Size-independent properties beyond the oracle-comparison sizes: NTT(delta_0) = 1,
    NTT(1) = n*delta_0, linearity, round trip."""
    py = pyoracle
    log_n = 22
    n = 1 << log_n
    one = oracle.int_to_limbs(py.to_mont(1, py.R))
    delta = np.zeros((n, 4), dtype=np.uint64)
    delta[0] = one
    assert (ctx.ntt(delta) == one).all()
    ones = np.tile(one, (n, 1))
    y = ctx.ntt(ones)
    assert oracle.limbs_to_int(y[0]) == py.to_mont(n, py.R) and not y[1:].any()
    x = oracle.splitmix_fr(0x1177, n, montgomery=True)
    fx = ctx.ntt(x)
    assert (ctx.ntt(fx, inverse=True) == x).all()
    # linearity on a sample of outputs: NTT(x + delta) = NTT(x) + 1
    xd = x.copy()
    xd[0] = oracle.fp_binop("orc_fp_add", oracle.FR, x[0], one)
    fxd = ctx.ntt(xd)
    for i in (0, 1, 12345, n - 1):
        assert (fxd[i] == oracle.fp_binop("orc_fp_add", oracle.FR, fx[i], one)).all()


def test_ntt_device_batch(ctx, oracle):
    import torch
    log_n, batch = 12, 5
    n = 1 << log_n
    x = oracle.splitmix_fr(0x2024, n * batch, montgomery=True).reshape(batch, n, 4)
    t = torch.from_numpy(x.view(np.int64).copy()).cuda()
    torch.cuda.synchronize()
    ctx.ntt_device(t.data_ptr(), log_n, inverse=False, coset=True, batch=batch, stride=n)
    got = t.cpu().numpy().view(np.uint64)
    for b in range(batch):
        assert (got[b] == oracle.ntt(x[b], coset=True)).all()


@pytest.mark.parametrize("log_n", [12, 21])
def test_ntt_device_batch_stride_padding(ctx, oracle, log_n):
    """Three transforms stride > n apart (a one-pass and a three-pass size, all four variants): each equals the oracle's,
    and every word of the padding after each transform — the three-pass transform goes through a scratch buffer laid
    out with the same stride — is left as it was."""
    import torch
    n, batch = 1 << log_n, 3
    stride = n + 37
    sentinel = np.uint64(0xA5A5A5A5A5A5A5A5)
    x = oracle.splitmix_fr(0x5791 + log_n, n * batch, montgomery=True).reshape(batch, n, 4)
    buf = np.full((batch, stride, 4), sentinel, dtype=np.uint64)
    buf[:, :n] = x
    for inverse, coset in VARIANTS:
        t = torch.from_numpy(buf.view(np.int64).copy()).cuda()
        torch.cuda.synchronize()
        ctx.ntt_device(t.data_ptr(), log_n, inverse=inverse, coset=coset, batch=batch, stride=stride)
        got = t.cpu().numpy().view(np.uint64)
        assert (got[:, n:] == sentinel).all(), (inverse, coset)
        for b in range(batch):
            assert (got[b, :n] == oracle.ntt(x[b], inverse=inverse, coset=coset)).all(), (log_n, b, inverse, coset)
