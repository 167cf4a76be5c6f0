"""The violation catalogue (tests/unsat_shapes.py) without a GPU: every case's claims hold, the oracle refuses every
violation and proves every control, and round 3's degree check, restated from plonk.cu's constants, misses exactly
the low-degree violations the catalogue says it misses — the reason the prover also checks its opening at zeta."""
import re

import numpy as np
import pytest

import unsat_shapes as us
from renegade_b200 import synth
from test_prove_witness_cpu import cycles
from witness_shapes import _source

R = synth.R
TAU = 0x1D2C3B4A59687706F5E4D3C2B1A09F8E7D6C5B4A39281706F5E4D3C2B1A0987
CASES = us.catalogue(10)


def _ints(a):
    return [int.from_bytes(np.ascontiguousarray(x).tobytes(), "little") * pow(2, -256, R) % R for x in a]


def test_domain_generator_is_the_oracles(oracle):
    for log_n in (2, 4, 10, 16):
        assert _ints([oracle.domain_generator(log_n)])[0] == us.omega(log_n)


@pytest.mark.parametrize("case", CASES, ids=[c.name for c in CASES])
def test_case_claims(case, oracle):
    n = case.n
    gates = [synth.gate_value([case.sel[s][j] for s in range(13)], [case.wires[c][j] for c in range(5)],
                              case.pub[j] if j < case.num_inputs else 0) for j in range(n)]
    assert gates == case.violation
    assert [j for j in range(n) if gates[j]] == sorted(case.rows)
    # copy constraints: equal values on every cycle of the wiring's permutation
    flat = [v for col in case.wires for v in col]
    perm = us.wiring_permutation(case.wire_vars)
    holds = all(len({flat[p] for p in cyc}) == 1 for cyc in cycles(perm))
    assert holds == case.copies_hold
    if case.witness is not None:  # the wiring path proves the same table and public inputs
        assert flat == [case.witness[int(v)] for v in np.asarray(case.wire_vars).reshape(-1)]
        assert case.pub == [case.witness[int(case.wire_vars[4, j])] for j in range(case.num_inputs)]
    # degree of the violation polynomial, by an inverse transform
    if any(gates):
        coeffs = _ints(oracle.ntt(synth.to_mont_array(gates), inverse=True))
        assert max(i for i, c in enumerate(coeffs) if c) == case.deg_r
        assert case.expect == us.UNSAT
    else:
        assert case.deg_r is None
    if case.kind.startswith("low degree"):
        assert case.deg_r == int(case.kind.split()[-1])


def _oracle_prove(oracle, pyoracle, case):
    sel, wires, pub, perm, k, bl = case.tables()
    tau = oracle.int_to_limbs(pyoracle.to_mont(TAU % R, R))
    srs = oracle.srs_from_tau(tau, case.n + 3)
    pk = oracle.plonk_preprocess(case.log_n, sel, perm, k, srs)
    rc, proof, _, _ = oracle.plonk_prove(case.log_n, case.num_inputs, k, pk, wires, pub, bl, srs)
    return rc, proof, (k, pk, pub, tau)


@pytest.mark.parametrize("case", CASES, ids=[c.name for c in CASES])
def test_oracle_refuses_every_violation(case, oracle, pyoracle):
    rc, proof, (k, pk, pub, tau) = _oracle_prove(oracle, pyoracle, case)
    assert rc == case.expect
    if rc == 0:
        assert oracle.plonk_verify_known_tau(case.log_n, case.num_inputs, k, pk, pub, proof, tau)


def test_oracle_proves_the_satisfied_fresh_output_circuit(oracle, pyoracle):
    for log_n in (2, 4, 5):
        case = us.satisfied(log_n)
        rc, proof, (k, pk, pub, tau) = _oracle_prove(oracle, pyoracle, case)
        assert rc == 0 and oracle.plonk_verify_known_tau(log_n, case.num_inputs, k, pk, pub, proof, tau)


# ---- round 3 restated ------------------------------------------------------------------------------------------------
G, = (int(x) for x in re.search(r"const fe g = fe_from_u32<Fr>\((\d+)\);", _source("plonk.cu")).groups())
assert re.search(r"const fe sj = FMUL\(g, host_pow\(w8n, \(uint64_t\)j\)\);", _source("plonk.cu")), \
    "the cosets are no longer s_j = g w_8n^j"


def _solve(a, b):
    """a x = b mod R (a square, invertible), by Gaussian elimination."""
    m = len(a)
    aug = [list(row) + [v] for row, v in zip(a, b)]
    for c in range(m):
        piv = next(r for r in range(c, m) if aug[r][c])
        aug[c], aug[piv] = aug[piv], aug[c]
        inv = pow(aug[c][c], -1, R)
        aug[c] = [x * inv % R for x in aug[c]]
        for r in range(m):
            if r != c and aug[r][c]:
                f = aug[r][c]
                aug[r] = [(x - f * y) % R for x, y in zip(aug[r], aug[c])]
    return [row[-1] for row in aug]


def round3_quotient(log_n, nc, r_coeffs):
    """What round 3 makes of a numerator r (coefficients, deg < n) that Z_H does not divide: the values r / Z_H on the
    nc cosets s_j H (s_j = g w_8n^j), one inverse transform per coset, un-scaled by s_j^-i, and the cosets un-mixed
    through the Vandermonde matrix in c_j = s_j^n (k_coset_combine).  Returns the nc n coefficients."""
    n = 1 << log_n
    w, w8n = us.omega(log_n), pow(5, (R - 1) // (8 * n), R)
    ninv = pow(n, -1, R)
    rows = []
    for j in range(nc):
        sj = G * pow(w8n, j, R) % R
        cj = pow(sj, n, R)
        zinv = pow(cj - 1, -1, R)
        vals = []
        for h in range(n):
            x = sj * pow(w, h, R) % R
            vals.append(sum(c * pow(x, i, R) for i, c in enumerate(r_coeffs)) * zinv % R)
        winv = pow(w, -1, R)
        coef = [sum(vals[h] * pow(winv, h * i, R) for h in range(n)) * ninv % R for i in range(n)]
        sinv = pow(sj, -1, R)
        rows.append((cj, [c * pow(sinv, i, R) % R for i, c in enumerate(coef)]))
    vand = [[pow(cj, k, R) for k in range(nc)] for cj, _ in rows]
    out = [0] * (nc * n)
    for i in range(n):  # coefficient i of each block q_k: sum_k c_j^k q_k[i] = coset j's coefficient i
        qk = _solve(vand, [coef[i] for _, coef in rows])
        for k in range(nc):
            out[k * n + i] = qk[k]
    return out


def round3_refuses(log_n, nc, r_coeffs):
    """k_check_degree's bit 0: a coefficient above NW (n + 1) + 2 is non-zero."""
    q = round3_quotient(log_n, nc, r_coeffs)
    return any(q[us.quotient_degree(log_n) + 1:])


@pytest.mark.parametrize("log_n", [2, 3, 4, 5])
def test_round3_degree_check_misses_exactly_degree_7_and_below(log_n):
    n, nc = 1 << log_n, us.cosets(log_n)
    assert nc == (6 if log_n >= 4 else 8)
    for d in range(n):
        r = [0] * d + [1]
        misses = not round3_refuses(log_n, nc, r)
        assert misses == us.degree_check_misses(log_n, d), d
        assert misses == (nc == 6 and d <= 7), d
    # a single-row violation (degree n - 1, every coefficient non-zero) is always caught
    lag = [pow(n, -1, R)] * n  # the Lagrange polynomial of row 0
    assert round3_refuses(log_n, nc, lag)


@pytest.mark.parametrize("log_n", [4, 5])
def test_seven_cosets_would_see_every_violation(log_n):
    n = 1 << log_n
    for d in range(n):
        assert round3_refuses(log_n, 7, [0] * d + [1]), d
