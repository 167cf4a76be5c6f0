"""Test infrastructure: the shapes where the collaborative prover (renegade_b200/collaborative.py) can go wrong, shared by
tests/test_collaborative_shapes_cpu.py (host backend) and tests/test_gpu_collaborative_shapes.py (device backend).

The joint prover interpolates its quotient from all 8 cosets of H (m = 8n, z(wX) = a roll by 8 of z on the coset
points), where the single prover switches to 6 cosets from n = 2^COSET_SWITCH on.  With 8 cosets the error term of a
violation polynomial r is X^(7n) r(X), above the degree bound 5n + 7 for every r != 0 once n >= 4: round 3's opened
tail refuses every unsatisfied witness (`quotient_blocks` restates the interpolation; the CPU test checks it).

The vector lengths its device primitives see cross kernel boundaries: m = 8n crosses the batch inversion's block of
kInvBlock elements, the wire polynomials (n + 2 coefficients) and z (n + 3) go through the CH-chunked Horner scans of
`b200_fr_poly_eval_device` / `b200_fr_poly_div_linear_device` at every level count.  The constants are read from
plonk.cu and collaborative.py, so the claims follow them if they move.

Share patterns: how a witness table (or the 17 blinders) is split between the parties.  Each returns one (rows, 4)
Montgomery-limb array per party whose sum mod r is the table."""
from __future__ import annotations

import os
import random
import re

import numpy as np
import pytest

import large_domains as ld
from renegade_b200 import _lib, synth
from witness_shapes import _constants

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
R = synth.R
NW = synth.N_WIRES
CH, = _constants("plonk.cu", r"constexpr int CH = (\d+);")
COSET_SWITCH, NC_LARGE, NC_SMALL = _constants("plonk.cu", r"const int nc = log_n >= (\d+) \? (\d+) : (\d+);")
INV_THREADS, INV_CHUNK = _constants("plonk.cu", r"constexpr int kInvThreads = (\d+), kInvChunk = (\d+), "
                                                r"kInvBlock = kInvThreads \* kInvChunk;")
INV_BLOCK = INV_THREADS * INV_CHUNK


def _collab_source() -> str:
    with open(os.path.join(ROOT, "renegade_b200", "collaborative.py")) as f:
        return f.read()


def _joint_cosets() -> int:
    src = _collab_source()
    m = re.search(r"m, log_m = (\d+) \* n, pk\.log_n \+ (\d+)", src)
    assert m, "collaborative.py no longer sets m, log_m = c * n, log_n + log c"
    cosets, log_c = int(m.group(1)), int(m.group(2))
    assert cosets == 1 << log_c
    roll = re.search(r"ce_zw = \[be\.roll\(v, (\d+)\) for v in ce_z\]", src)
    assert roll and int(roll.group(1)) == cosets, "z(w x) is no longer a roll by the coset count"
    return cosets


JOINT_COSETS = _joint_cosets()


def quotient_bound(n: int) -> int:
    """Round 3's bound: the quotient's top coefficient NW (n + 1) + 2 (= 5n + 7)."""
    return NW * (n + 1) + 2


def levels(length: int) -> int:
    """Kernel levels of the CH-chunked Horner scans (`eval_batch`, `horner_suffix`): chunks of CH, then chunks of the
    chunk totals, ... down to one."""
    lv, n = 1, length
    while n > CH:
        n = (n + CH - 1) // CH
        lv += 1
    return lv


# ---- round 3 of the joint prover, restated ------------------------------------------------------------------------------
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


def quotient_blocks(log_n: int, nc: int, g: int = 5) -> list:
    """The interpolated quotient of r = X^d over nc cosets s_j H (s_j = g w_8n^j), for any d < n.  On s_j H, X^n is the
    constant c_j = s_j^n, so r / Z_H takes the values X^d / (c_j - 1) there.  Writing the quotient of degree < nc n as
    sum_k X^(kn) q_k(X) with deg q_k < n, it agrees with those values on coset j exactly when sum_k c_j^k q_k = X^d /
    (c_j - 1) as polynomials of degree < n: q_k = a_k X^d with sum_k c_j^k a_k = 1 / (c_j - 1).  Returns the a_k — the
    quotient's coefficient k n + d is a_k, every other coefficient is zero (whatever d is)."""
    n = 1 << log_n
    w8n = pow(5, (R - 1) // (8 * n), R)
    c = [pow(g * pow(w8n, j, R) % R, n, R) for j in range(nc)]
    return _solve([[pow(cj, k, R) for k in range(nc)] for cj in c], [pow(cj - 1, -1, R) for cj in c])


def round3_refuses_monomial(log_n: int, nc: int, d: int) -> bool:
    """Whether the interpolated quotient of r = X^d has a non-zero coefficient in [5n + 8, nc n): what round 3's opened
    tail (`tail[0] == 0 or any(tail[1:])`, the tail starting at 5n + 7) sees of a violation X^d."""
    n = 1 << log_n
    a = quotient_blocks(log_n, nc)
    return any(a[k] for k in range(nc) if quotient_bound(n) < k * n + d < nc * n)


# ---- buffer sizes of the device primitives, restated from plonk.cu --------------------------------------------------------
def _check_reserves():
    src = ld.plonk_source()
    assert re.search(r"const size_t L = len \+ 8;\s*int rc = ctx->c\.plonk_ws\.reserve\(\(L \+ 4 \* \(L / CH \+ 4 \* CH \+ 64\)"
                     r" \+ 16\) \* sizeof\(fe\)\);", src), "b200_fr_poly_div_linear_device's reserve changed: restate it here"
    assert re.search(r"int rc = ctx->c\.ntt_scratch\.reserve\(n \* sizeof\(fe\)\);\s*if \(rc != B200_OK\) return rc;\s*"
                     r"batch_inverse_enqueue", src), "b200_fr_batch_inverse_device's reserve changed: restate it here"
    assert re.search(r"bf\.ws->reserve\(workspace_elems\(n, k\) \* sizeof\(fe\)\)", src)


_check_reserves()
PLONK = ld.constants()


def div_linear_ws_elems(length: int) -> int:
    """plonk_ws elements `b200_fr_poly_div_linear_device` reserves for a polynomial of `length` coefficients."""
    L = length + 8
    return L + 4 * (L // CH + 4 * CH + 64) + 16


def joint_ws_elems(log_n: int) -> int:
    """The most plonk_ws a joint proof reserves: its divisions are of n + 3 coefficients (the batched polynomial and z)."""
    return div_linear_ws_elems((1 << log_n) + 3)


def joint_inverse_elems(log_n: int) -> int:
    """The most NTT scratch a joint proof reserves: the batch inversion of 1 / (n (x - 1)) over the m = 8n coset points."""
    return JOINT_COSETS << log_n


def prover_ws_elems(log_n: int) -> int:
    """plonk_ws elements a single proof of a 2^log_n key reserves (the prover's workspace carve, one proof)."""
    return ld.workspace_elems(1 << log_n, 1, PLONK)


def prover_ntt_scratch_elems(log_n: int) -> int:
    """NTT scratch elements a key and its single proofs reserve: NS m from preprocess, 7 m per table proof."""
    m = ld.cosets(log_n, PLONK) << log_n
    return max(PLONK["NS"] * m, PLONK["STAGE_PER_M"] * m)


def circuit(log_n: int, num_inputs, seed: int = 300):
    """A satisfied synth circuit with `num_inputs` public inputs (at most n - 1: at 2^2, 3), or with every row public
    (num_inputs = "all": witness_shapes.every_row_public, its permutation derived from the wiring)."""
    import dataclasses
    if num_inputs == "all":
        from test_prove_witness_cpu import wiring_permutation
        from witness_shapes import every_row_public
        c = every_row_public(log_n).circ
        return dataclasses.replace(c, perm=wiring_permutation(c.wire_vars))
    return synth.synth_circuit(log_n, num_inputs=min(num_inputs, (1 << log_n) - 1), seed=seed + log_n, check=log_n <= 10)


# ---- share patterns ---------------------------------------------------------------------------------------------------
def ints(arr) -> list:
    return synth_ints(np.asarray(arr, dtype=np.uint64).reshape(-1, 4))


def synth_ints(a) -> list:
    rinv = pow(2, -256, R)
    return [int.from_bytes(np.ascontiguousarray(x).tobytes(), "little") * rinv % R for x in a]


def mont(vals) -> np.ndarray:
    return synth.to_mont_array([v % R for v in vals]).reshape(-1, 4)


PATTERNS = {"random": (2, 3), "zero_party0": (2, 3), "equal": (2, 3), "minus_one": (2,), "cancel": (3,)}


def share(values, parties: int, pattern: str = "random", seed: int = 0) -> list:
    """Split a (rows, 4) Montgomery table t into `parties` additive shares:
      random       seeded random shares (`collaborative.share_table`);
      zero_party0  party 0 holds all zeros (its commitments are identity records), the others a random split of t;
      equal        every party holds t / parties (every opened commitment is a sum of equal points: a doubling);
      minus_one    (r - 1, t + 1);
      cancel       (s, -s, t): the first two parties' shares cancel."""
    from renegade_b200 import collaborative as co
    assert pattern == "random" or parties in PATTERNS[pattern], (pattern, parties)
    t = ints(values)
    rows = len(t)
    if pattern == "random":
        return co.share_table(mont(t), parties, seed)
    if pattern == "zero_party0":
        rest = co.share_table(mont(t), parties - 1, seed)
        return [mont([0] * rows)] + rest
    if pattern == "equal":
        inv = pow(parties, -1, R)
        return [mont([v * inv for v in t]) for _ in range(parties)]
    if pattern == "minus_one":
        return [mont([R - 1] * rows), mont([v + 1 for v in t])]
    rnd = random.Random(seed)
    s = [rnd.randrange(1, R) for _ in range(rows)]
    return [mont(s), mont([-x for x in s]), mont(t)]


def summed(shares) -> list:
    """The table the shares stand for, with Python integers."""
    cols = [ints(s) for s in shares]
    return [sum(c) % R for c in zip(*cols)]


def nonzero_blinder_split(blinders, parties: int, seed: int) -> list:
    """Random shares of the 17 blinders in which every party's share of every blinder is non-zero (so a zero blinder
    is zero only in the sum)."""
    t = ints(blinders)
    rnd = random.Random(seed)
    while True:
        sh = [[rnd.randrange(1, R) for _ in t] for _ in range(parties - 1)]
        last = [(v - sum(col)) % R for v, col in zip(t, zip(*sh))]
        if all(last):
            return [mont(s) for s in sh] + [mont(last)]


# ---- the violation catalogue ------------------------------------------------------------------------------------------------
def catalogue_case(oracle, tau, case, prove_joint):
    """Run one case of tests/unsat_shapes.py through `prove_joint(sel, perm, k, wires, pub, wire_shares, bl_shares) ->
    proof` with 2 parties, the blinders split so that every party's share of every blinder is non-zero (a zeroed
    blinder is zero only in the sum).  expect == UNSAT must raise B200_ERR_UNSATISFIED and is followed by the case's
    satisfying control on the same backend; the control and every expect == 0 case must give the oracle's bytes."""
    import unsat_shapes as us
    sel, wires, pub, perm, k, bl = case.tables()
    srs = oracle.srs_from_tau(tau, case.n + 3)
    opk = oracle.plonk_preprocess(case.log_n, sel, perm, k, srs)
    ws = share(wires.reshape(-1, 4), 2, "random", seed=case.log_n * 31 + len(case.name))
    bs = nonzero_blinder_split(bl, 2, seed=len(case.name))
    if case.expect == us.UNSAT:
        with pytest.raises(_lib.B200Error) as err:
            prove_joint(sel, perm, k, wires, pub, ws, bs)
        assert err.value.code == _lib.B200_ERR_UNSATISFIED, case.name
        gw, gp = case.good
        wires = np.stack([synth.to_mont_array(c) for c in gw])
        pub = synth.to_mont_array(gp).reshape(-1, 4)
        ws = share(wires.reshape(-1, 4), 2, "random", seed=7)
        bl = synth.to_mont_array([0x51 + i for i in range(17)])
        bs = nonzero_blinder_split(bl, 2, seed=8)
    rc, oproof, _, _ = oracle.plonk_prove(case.log_n, case.num_inputs, k, opk, wires, pub, bl, srs)
    assert rc == 0
    proof = prove_joint(sel, perm, k, wires, pub, ws, bs)
    assert bytes(proof) == bytes(oproof), case.name


# ---- what the parties open ---------------------------------------------------------------------------------------------------
def opened_vectors(monkeypatch, run):
    """Run `run()` with `collaborative.Fabric` replaced by a subclass that records every opened vector (as integers)."""
    from renegade_b200 import collaborative as co
    seen = []

    class Recording(co.Fabric):
        def open(self, x):
            acc = super().open(x)
            seen.append(ints(self.be.to_limbs(acc)))
            return acc

    monkeypatch.setattr(co, "Fabric", Recording)
    return run(), seen


def z_over_h(circ, beta: int, gamma: int) -> list:
    """The permutation product on H with Python integers: z(w^0) = 1, z(w^(j+1)) = z(w^j) prod_i (w_i + beta k_i w^j +
    gamma) / (w_i + beta sigma_i(w^j) + gamma), sigma_i(w^j) = k_(perm / n) w^(perm mod n)."""
    n = circ.n
    w = pow(5, (R - 1) >> circ.log_n, R)
    k = ints(circ.k)
    wires = ints(circ.wires)
    perm = [int(x) for x in np.asarray(circ.perm).reshape(-1)]
    dom = [pow(w, j, R) for j in range(n)]
    z = [1]
    for j in range(n - 1):
        num = den = 1
        for i in range(NW):
            v = wires[i * n + j]
            t = perm[i * n + j]
            num = num * (v + beta * k[i] * dom[j] + gamma) % R
            den = den * (v + beta * k[t // n] * dom[t % n] + gamma) % R
        z.append(z[-1] * num * pow(den, -1, R) % R)
    return z


def _contains_run(vec, col) -> bool:
    n = len(col)
    first = col[0]
    return any(vec[i] == first and vec[i:i + n] == col for i in range(len(vec) - n + 1))


def check_openings(circ, hint, seen, challenges, ntt):
    """No opened vector contains a wire column of the summed table or z's evaluations over H as a contiguous run, except
    two documented openings: the hint's blinded wire-0 polynomial (opened for the linking hint; folded mod X^n - 1 it is
    wire 0 on H, which `ntt` — a forward transform of n integers — shows) and round 3's tail (the last vector
    opened: coefficients 5n + 7 … 8n - 1 of the quotient, the top one non-zero, the others zero)."""
    n = circ.n
    table = ints(circ.wires)
    cols = [table[i * n:(i + 1) * n] for i in range(NW)]
    beta, gamma = (synth_ints(np.asarray(getattr(challenges, f), dtype=np.uint64).reshape(1, 4))[0] for f in ("beta", "gamma"))
    z = z_over_h(circ, beta, gamma)
    link = ints(hint.linking_wire_poly)
    assert seen.count(link) == 1
    assert seen[-1][0] and not any(seen[-1][1:]) and len(seen[-1]) == JOINT_COSETS * n - quotient_bound(n)
    folded = [(link[i] + (link[i + n] if i + n < len(link) else 0)) % R for i in range(n)]
    assert ntt(folded) == cols[0]
    rest = [v for v in seen[:-1] if v != link]
    for target, what in [(c, f"wire {i}") for i, c in enumerate(cols)] + [(z, "z on H"), (z[1:], "z on H, shifted")]:
        if len(set(target)) == 1:
            continue  # a constant column (the zero variable) is no secret, and any run of equal values would match it
        for idx, v in enumerate(rest):
            assert not _contains_run(v, target), (what, idx)
