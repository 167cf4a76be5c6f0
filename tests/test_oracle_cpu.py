"""CPU tests: pin the oracle (C restatement) against the committed golden fixtures — the
reference-owned SRS bytes and the known answers from the independent big-int restatement —
and against the Python restatement on seeded inputs."""
import numpy as np
import pytest


def H(s):
    return int(s, 16)


def pt_to_mont(py, P):
    return np.frombuffer(py.encode_g1_mont(P), dtype=np.uint64).copy()


def test_constants(oracle, pyoracle, kat):
    py = pyoracle
    assert H(kat["fr_modulus"]) == py.R and H(kat["fq_modulus"]) == py.Q
    one = np.array([1, 0, 0, 0], dtype=np.uint64)
    for which, mod, key in ((oracle.FR, py.R, "fr"), (oracle.FQ, py.Q, "fq")):
        r1 = oracle.limbs_to_int(oracle.fp_unop("orc_fp_to_mont", which, one))
        assert r1 == H(kat[key + "_R"]) == (1 << 256) % mod
        # R^2 = to_mont(to_mont(1))
        r2 = oracle.limbs_to_int(oracle.fp_unop("orc_fp_to_mont", which, oracle.int_to_limbs(r1)))
        assert r2 == H(kat[key + "_R2"])
    w = oracle.limbs_to_int(oracle.fp_unop("orc_fp_from_mont", oracle.FR, oracle.domain_generator(28)))
    assert w == H(kat["fr_root_2_28"])
    assert pow(w, 1 << 28, py.R) == 1 and pow(w, 1 << 27, py.R) != 1


def test_field_mul_kat(oracle, pyoracle, kat):
    py = pyoracle
    for rec in kat["field_mul"]:
        which, mod = (oracle.FR, py.R) if rec["field"] == "fr" else (oracle.FQ, py.Q)
        a, b = H(rec["a"]), H(rec["b"])
        am, bm = oracle.int_to_limbs(py.to_mont(a, mod)), oracle.int_to_limbs(py.to_mont(b, mod))
        got = oracle.limbs_to_int(oracle.fp_binop("orc_fp_mul", which, am, bm))
        assert py.from_mont(got, mod) == H(rec["ab"])
        inv = oracle.limbs_to_int(oracle.fp_unop("orc_fp_inv", which, am))
        assert py.from_mont(inv, mod) == H(rec["a_inv"])


def test_srs_fixture_on_curve(oracle, pyoracle, kat, srs_head):
    """Reference-owned data: every committed SRS record is on the curve under the oracle's
    Fq / Montgomery arithmetic (the check srs.rs:178-179 makes), and decodes to the points the
    big-int restatement decodes."""
    py = pyoracle
    raw, n = py.parse_ptau_g1(srs_head + bytes(64 * (py.MAX_SRS_DEGREE + 1)), 512)
    pts = np.frombuffer(raw, dtype=np.uint64).reshape(-1, 8)
    assert pts.shape[0] == 512
    for i in range(512):
        assert oracle.g1_on_curve(pts[i])
    for i, exp in enumerate(kat["srs_points_0_3"]):
        assert py.decode_g1_mont(raw, i) == (H(exp[0]), H(exp[1]))
    assert py.decode_g1_mont(raw, 0) == (1, 2)  # tau^0 * G
    bad = pts[3].copy()
    bad[0] ^= np.uint64(1)
    assert not oracle.g1_on_curve(bad)


def test_g1_kat(oracle, pyoracle, kat):
    py = pyoracle
    g = pt_to_mont(py, py.G1_GEN)
    for k, key in ((2, "g1_2G"), (3, "g1_3G")):
        out, inf = oracle.g1_mul(g, False, oracle.int_to_limbs(k))
        assert not inf and py.decode_g1_mont(out.tobytes(), 0) == (H(kat[key][0]), H(kat[key][1]))
    e = kat["edge"]
    P = (H(e["P"][0]), H(e["P"][1]))
    Pm = pt_to_mont(py, P)
    out, inf = oracle.g1_add(Pm, False, Pm, False)
    assert py.decode_g1_mont(out.tobytes(), 0) == (H(e["P_plus_P"][0]), H(e["P_plus_P"][1]))
    out, inf = oracle.g1_add(Pm, False, pt_to_mont(py, (H(e["neg_P"][0]), H(e["neg_P"][1]))), False)
    assert inf
    out, inf = oracle.g1_mul(Pm, False, oracle.int_to_limbs(py.R - 1))
    assert py.decode_g1_mont(out.tobytes(), 0) == (H(e["r_minus_1_times_P"][0]), H(e["r_minus_1_times_P"][1]))


def test_msm_known_dlog_kat(oracle, pyoracle, kat):
    py = pyoracle
    for rec in kat["msm_known_dlog"]:
        n = rec["n"]
        bases = oracle.known_dlog_bases(0xB200, n)
        scalars = oracle.splitmix_fr(0x5CA1A8, n, montgomery=False)
        for naive in (False, True):
            out, inf = oracle.msm(bases, scalars, naive=naive)
            assert not inf
            assert py.decode_g1_mont(out.tobytes(), 0) == (H(rec["result"][0]), H(rec["result"][1]))


def test_msm_srs_kat(oracle, pyoracle, kat, srs_head):
    py = pyoracle
    pts = np.frombuffer(srs_head[80:80 + 64 * 16], dtype=np.uint64).reshape(16, 8)
    s = oracle.ints_to_array([H(v) for v in kat["msm_srs16"]["scalars"]])
    out, inf = oracle.msm(pts, s)
    exp = kat["msm_srs16"]["result"]
    assert py.decode_g1_mont(out.tobytes(), 0) == (H(exp[0]), H(exp[1]))


def test_msm_edge_cases(oracle, pyoracle):
    py = pyoracle
    n = 40
    bases = oracle.known_dlog_bases(0xB200, n)
    zeros = np.zeros((n, 4), dtype=np.uint64)
    out, inf = oracle.msm(bases, zeros)
    assert inf
    # duplicate points with cancelling scalars: s*P + (r-s)*P = identity
    dup = np.repeat(bases[:1], 2, axis=0)
    s = 0x1234567
    out, inf = oracle.msm(dup, oracle.ints_to_array([s, py.R - s]))
    assert inf
    # scalar r-1 on every point == negated sum
    sc = oracle.ints_to_array([py.R - 1] * n)
    out, inf = oracle.msm(bases, sc)
    a = py.splitmix_fr(0xB200, n)
    assert py.decode_g1_mont(out.tobytes(), 0) == py.g1_mul(py.G1_GEN, (-sum(a)) % py.R)
    # window rule of ark-ec 0.4.2 (SURVEY.md §8(a4))
    assert [oracle.msm_window_bits(v) for v in (31, 1 << 12, 1 << 16, (1 << 17) + 3, 1 << 20, 1 << 24)] == \
        [3, 10, 13, 14, 15, 18]


def test_ntt_kat(oracle, pyoracle, kat):
    py = pyoracle
    for rec in kat["ntt"]:
        x = [H(v) for v in rec["x"]]
        xm = oracle.ints_to_array([py.to_mont(v, py.R) for v in x])
        for key, inv, cos in (("fft", False, False), ("ifft", True, False), ("coset_fft", False, True)):
            y = oracle.ntt(xm, inverse=inv, coset=cos)
            got = [py.from_mont(v, py.R) for v in oracle.array_to_ints(y)]
            assert got == [H(v) for v in rec[key]], (rec["log_n"], key)


@pytest.mark.parametrize("log_n", [0, 1, 5, 9, 12])
def test_ntt_properties(oracle, pyoracle, log_n):
    py = pyoracle
    n = 1 << log_n
    x = oracle.splitmix_fr(0x1177, n, montgomery=True)
    for cos in (False, True):
        assert (oracle.ntt(oracle.ntt(x, False, cos), True, cos) == x).all()
    # NTT(delta_0) = all ones ; NTT(all ones) = n * delta_0
    one = oracle.int_to_limbs(py.to_mont(1, py.R))
    delta = np.zeros((n, 4), dtype=np.uint64)
    delta[0] = one
    assert (oracle.ntt(delta) == np.tile(one, (n, 1))).all()
    y = oracle.ntt(np.tile(one, (n, 1)))
    assert oracle.limbs_to_int(y[0]) == py.to_mont(n % py.R, py.R) and not y[1:].any()
    if log_n <= 9:
        xi = [py.from_mont(v, py.R) for v in oracle.array_to_ints(x)]
        assert [py.from_mont(v, py.R) for v in oracle.array_to_ints(oracle.ntt(x))] == py.ntt(xi)


def test_splitmix_and_bases_match_python(oracle, pyoracle):
    py = pyoracle
    assert oracle.array_to_ints(oracle.splitmix_fr(0x5CA1A8, 50, False)) == py.splitmix_fr(0x5CA1A8, 50)
    assert oracle.array_to_ints(oracle.splitmix_fr(0x5CA1A8, 5, False, first=45)) == py.splitmix_fr(0x5CA1A8, 50)[45:]
    B = oracle.known_dlog_bases(0xB200, 6)
    a = py.splitmix_fr(0xB200, 6)
    for i in range(6):
        assert py.decode_g1_mont(B.tobytes(), i) == py.g1_mul(py.G1_GEN, a[i])


@pytest.mark.parametrize("n, first_a, first_b", [(0, 0, 0), (1, 0, 0), (5, (1 << 26) - 5, (1 << 26) - 5),
                                                  ((1 << 14) - 1, 0, 7), ((1 << 14) + 1, 3, 0), (1 << 16, 0, 1 << 22)])
def test_fr_dot_matches_python(oracle, pyoracle, n, first_a, first_b):
    """orc_fr_dot, the closed form of the large known-dlog MSMs, against Python integers: across its chunk edges
    (2^14 terms) and at the offsets the GPU tests use (the top 5 of 2^26 bases, batch members 2^22 scalars apart)."""
    a = oracle.array_to_ints(oracle.splitmix_fr(0xB200, n, False, first=first_a))
    b = oracle.array_to_ints(oracle.splitmix_fr(0x5CA1A8, n, False, first=first_b))
    assert oracle.fr_dot(0xB200, 0x5CA1A8, n, first_a, first_b) == sum(x * y for x, y in zip(a, b)) % pyoracle.R


def test_quotient_domain_of_six_cosets_matches_the_8n_coset(pyoracle):
    """The algebra behind the device prover's quotient domain (DESIGN.md §4), pinned with the Python oracle's own
    transforms: a polynomial t of degree <= 5n + 7 is recovered from its values on 6 of the 8 cosets s_j * H_n of
    g * H_8n (the reference's quotient domain) by 6 size-n inverse transforms, the scaling s_j^-i and one 6 x 6
    inverse-Vandermonde combination in c_j = s_j^n — and a polynomial with n + 3 coefficients is evaluated on coset j
    by folding X^n -> c_j, scaling by s_j^i and ONE size-n transform."""
    import random
    py = pyoracle
    rnd = random.Random(0xC05E7)
    log_n, nc = 4, 6
    n, g = 1 << log_n, py.FR_GENERATOR
    w8n = py.domain_generator(log_n + 3)
    s = [g * pow(w8n, j, py.R) % py.R for j in range(nc)]
    c = [pow(sj, n, py.R) for sj in s]
    t = [rnd.randrange(py.R) for _ in range(5 * n + 8)] + [0] * (8 * n - (5 * n + 8))
    on_8n = py.coset_ntt(t)  # what the reference computes: t on g * w_8n^i, natural order
    # coset j of the 8n domain is every 8th point starting at j
    vals = [[on_8n[8 * h + j] for h in range(n)] for j in range(nc)]
    u = []
    for j in range(nc):
        v = py.ntt(vals[j], inverse=True)  # coefficients of u_j(s_j X)
        u.append([v[i] * pow(s[j], -i, py.R) % py.R for i in range(n)])
    # invert the Vandermonde matrix V[j][k] = c_j^k by Gauss-Jordan
    m = [[pow(c[j], k, py.R) for k in range(nc)] + [int(i == j) for i in range(nc)] for j in range(nc)]
    for col in range(nc):
        piv = next(r for r in range(col, nc) if m[r][col])
        m[col], m[piv] = m[piv], m[col]
        inv = pow(m[col][col], -1, py.R)
        m[col] = [x * inv % py.R for x in m[col]]
        for r in range(nc):
            if r != col and m[r][col]:
                f = m[r][col]
                m[r] = [(x - f * y) % py.R for x, y in zip(m[r], m[col])]
    minv = [row[nc:] for row in m]
    rec = [sum(minv[k][j] * u[j][i] for j in range(nc)) % py.R for k in range(nc) for i in range(n)]
    assert rec == t[:nc * n]
    # forward direction: fold + scale + size-n transform == the 8n-coset values on that coset
    a = [rnd.randrange(py.R) for _ in range(n + 3)]
    a_on_8n = py.coset_ntt(a + [0] * (8 * n - len(a)))
    for j in range(nc):
        folded = [(a[i] + (c[j] * a[n + i] if n + i < len(a) else 0)) * pow(s[j], i, py.R) % py.R for i in range(n)]
        assert py.ntt(folded) == [a_on_8n[8 * h + j] for h in range(n)], j


def test_oracle_prover_reproduces_the_committed_proof():
    """tests/golden/proof_kat.json: proof bytes, Fiat-Shamir challenges, verifying key and linking polynomial of one seeded
    circuit as the oracle prover produced them when the fixture was cut (tests/golden/make_proof_golden.py).  A regression
    pin of the restated rounds / transcript / blinding order — not a vector of the Rust reference (DESIGN.md section 5).
    tests/test_gpu_plonk.py compares the device proof with the same bytes."""
    import json
    import os
    import sys
    here = os.path.dirname(os.path.abspath(__file__))
    sys.path.insert(0, os.path.join(here, "golden"))
    import make_proof_golden
    with open(os.path.join(here, "golden", "proof_kat.json")) as f:
        want = json.load(f)
    assert make_proof_golden.compute(want["params"]) == want
