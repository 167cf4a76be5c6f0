"""Test infrastructure: Poseidon2 (t = 3) states built to reach reduction edges, restated with Python integers.

The device kernels work on Montgomery residues (a value v is stored as v * 2^256 mod r), so every edge here is a
RESIDUE: what the kernel's adds and products see.  `mont(v)` / `unmont(w)` convert; the forward and inverse rounds run
on plain values, like bn254_py.poseidon2_permute.

x -> x^5 is a bijection of Fr (gcd(5, r - 1) = 1), M_E = circ(2, 1, 1) has determinant 4 and M_I = [[2,1,1],[1,2,1],
[1,1,3]] determinant 7, so the permutation runs backwards: `inverse_from(round, state)` undoes the rounds before
`round` (inverse S-box x^(5^-1 mod (r - 1)), inverse MDS matrices, round constants subtracted).  `targeted_states`
uses it to build states whose S-box input at a chosen round and lane is a chosen residue; `forward_sbox_inputs`
runs the forward permutation recording every S-box input, so each state's claim is checked, not assumed.

Rounds are numbered as they run: 0..3 the first full rounds, 4..59 the 56 partial rounds, 60..63 the last full
rounds."""
from __future__ import annotations

import random

from field_edges import MONT, R_FR, operands

R = R_FR
N_ROUNDS = 64
FULL_FIRST, PARTIAL, FULL_LAST = range(0, 4), range(4, 60), range(60, 64)
SBOX_INV = pow(5, -1, R - 1)
M_E = [[2, 1, 1], [1, 2, 1], [1, 1, 2]]
M_I = [[2, 1, 1], [1, 2, 1], [1, 1, 3]]

# S-box input targets (residues): zero, the residue one, r - 1, (r -+ 1) / 2, the field's one (R mod r) and 2^253
TARGETS = [0, 1, R - 1, (R - 1) // 2, (R + 1) // 2, MONT % R, 1 << 253]
# the (round, lane) positions targeted: every full round and lane, and the first, a middle and the last partial round
POSITIONS = [(rd, lane) for rd in (*FULL_FIRST, *FULL_LAST) for lane in range(3)] + [(4, 0), (31, 0), (59, 0)]


def mont(v: int) -> int:
    return v * MONT % R


def unmont(w: int) -> int:
    return w * pow(MONT, -1, R) % R


def _mat_vec(m, v):
    return [sum(m[i][j] * v[j] for j in range(3)) % R for i in range(3)]


def _mat_inv(m):
    """Inverse of a 3 x 3 matrix mod r by the adjugate."""
    cof = [[(m[(i + 1) % 3][(j + 1) % 3] * m[(i + 2) % 3][(j + 2) % 3] -
             m[(i + 1) % 3][(j + 2) % 3] * m[(i + 2) % 3][(j + 1) % 3]) for j in range(3)] for i in range(3)]
    det = sum(m[0][j] * cof[0][j] for j in range(3)) % R
    d = pow(det, -1, R)
    return [[cof[j][i] * d % R for j in range(3)] for i in range(3)]  # transpose of the cofactors


M_E_INV, M_I_INV = _mat_inv(M_E), _mat_inv(M_I)


def _rc(full, partial, rd, lane):
    if rd in PARTIAL:
        return partial[rd - 4] if lane == 0 else 0
    return full[3 * (rd if rd < 4 else rd - 56) + lane]


def _round(st, rd, full, partial, hook=None):
    lanes = range(1) if rd in PARTIAL else range(3)
    st = list(st)
    for i in lanes:
        x = (st[i] + _rc(full, partial, rd, i)) % R
        if hook:
            hook(rd, i, x)
        st[i] = pow(x, 5, R)
    return _mat_vec(M_I if rd in PARTIAL else M_E, st)


def _round_inv(st, rd, full, partial):
    st = _mat_vec(M_I_INV if rd in PARTIAL else M_E_INV, st)
    for i in (range(1) if rd in PARTIAL else range(3)):
        st[i] = (pow(st[i], SBOX_INV, R) - _rc(full, partial, rd, i)) % R
    return st


def forward_sbox_inputs(state, full, partial):
    """(output, {(round, lane): S-box input}) of the permutation of `state` (plain values)."""
    seen = {}
    st = _mat_vec(M_E, state)
    for rd in range(N_ROUNDS):
        st = _round(st, rd, full, partial, hook=lambda r, i, x: seen.__setitem__((r, i), x))
    return st, seen


def inverse_from(rd, st, full, partial):
    """The input state whose state just before round `rd` is `st` (plain values)."""
    for k in reversed(range(rd)):
        st = _round_inv(st, k, full, partial)
    return _mat_vec(M_E_INV, st)


def targeted_states(full, partial, seed=0x9052):
    """[(round, lane, target residue, input state as residues)]: the S-box input of that lane in that round is the
    target residue; the other lanes of the state before that round are seeded random values."""
    rng = random.Random(seed)
    out = []
    for rd, lane in POSITIONS:
        for t in TARGETS:
            st = [rng.randrange(R) for _ in range(3)]
            st[lane] = (unmont(t) - _rc(full, partial, rd, lane)) % R
            out.append((rd, lane, t, [mont(v) for v in inverse_from(rd, st, full, partial)]))
    return out


def edge_states(seed=0xED6E):
    """[(label, state as residues)]: one lane an edge operand and the others 0, (v, v, v) for every operand (with
    (r - 1, r - 1, r - 1) the external MDS sum 3(r - 1) wraps twice), and states whose first external MDS output is
    exactly 0 or r - 1 in one lane."""
    ops = operands(R)
    out = []
    for lane in range(3):
        for v in ops:
            s = [0, 0, 0]
            s[lane] = v
            out.append((f"lane{lane}={v:#x}", s))
    out += [(f"all={v:#x}", [v, v, v]) for v in ops]
    rng = random.Random(seed)
    for lane in range(3):
        for t in (0, R - 1):
            for _ in range(4):
                y = [rng.randrange(R) for _ in range(3)]
                y[lane] = t
                out.append((f"mds0[{lane}]={t:#x}", _mat_vec(M_E_INV, y)))  # M_E is linear: residues map to residues
    return out


def external_mds(s):
    return _mat_vec(M_E, s)
