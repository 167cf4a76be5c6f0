"""Test infrastructure: witnesses that do NOT satisfy their circuit, at the shapes where refusing them can go wrong.

The prover refuses a witness (B200_ERR_UNSATISFIED, the reference's WrongQuotientPolyDegree) when round 3's quotient
has the wrong degree (`k_check_degree`) or when the batched polynomial opened at zeta does not take the value the
verifier expects (the self-check at the end of round 5).  The quotient is interpolated from NC_LARGE = 6 cosets of H
from n = 2^COSET_SWITCH on, from all 8 below.  Let r be the polynomial whose values on H are the per-row gate
violations: six cosets return the true quotient plus u(X^n) r(X) with deg u = 5, which stays under the allowed degree
5n + 7 exactly when deg r <= 7 ("low degree d" cases below).  Round 3 misses those; the self-check refuses them.

Most cases live on a "fresh-output" circuit: every row has q_o = 1 and q_c = c_i, w4 is a variable used on that row
only, w0..w3 are the zero variable (public rows: q_c = 0, w4 = the public input).  Shifting w4 on row i by -p(w^i)
makes row i's gate value p(w^i) and leaves every copy constraint holding.  Optional blank rows (every selector zero)
and shared variables on the wires the selectors ignore carry the copy-only cases.

Each builder returns a `Case`: the tables (ints; `tables()` gives the prover's Montgomery arrays), the wiring and a
witness vector where the case can be given as one (a witness vector cannot break a copy constraint, nor a public
input), the rows it claims are violated, the violation vector on H, whether the copy constraints hold, its class, and
the status the oracle (8n-point quotient, exact) must return.  tests/test_unsat_shapes_cpu.py checks every claim."""
from __future__ import annotations

import random
import re
from dataclasses import dataclass, field

import numpy as np

from renegade_b200 import synth
from test_prove_witness_cpu import wiring_permutation
from witness_shapes import _constants, _k, _source

R = synth.R
NW = synth.N_WIRES
CH, = _constants("plonk.cu", r"constexpr int CH = (\d+);")
COSET_SWITCH, NC_LARGE, NC_SMALL = _constants("plonk.cu", r"const int nc = log_n >= (\d+) \? (\d+) : (\d+);")
assert re.search(r"const size_t deg = NW \* \(n \+ 1\) \+ 2;", _source("plonk.cu")), \
    "round 3's degree bound is no longer NW (n + 1) + 2"
UNSAT = 2  # the oracle's refusal (WrongQuotientPolyDegree)


def quotient_degree(log_n: int) -> int:
    """Round 3's bound: the quotient's top coefficient, NW (n + 1) + 2."""
    return NW * ((1 << log_n) + 1) + 2


def omega(log_n: int) -> int:
    """Generator of H (5 generates Fr*; the device's and the oracle's domains use 5^((r - 1) / n))."""
    return pow(5, (R - 1) >> log_n, R)


def cosets(log_n: int) -> int:
    return NC_LARGE if log_n >= COSET_SWITCH else NC_SMALL


def degree_check_misses(log_n: int, deg_r: int) -> bool:
    """Whether round 3's degree check, on its nc cosets, passes a witness whose violation polynomial has degree deg_r:
    the error term u(X^n) r(X) has degree (nc - 1) n + deg_r (tests/test_unsat_shapes_cpu.py restates the interpolation
    and checks this rule)."""
    nc = cosets(log_n)
    return nc < 8 and (nc - 1) * (1 << log_n) + deg_r <= quotient_degree(log_n)


@dataclass
class Case:
    name: str
    log_n: int
    num_inputs: int
    sel: list                 # 13 x n ints
    wires: list               # 5 x n ints: the table the table path proves
    pub: list                 # num_inputs ints
    wire_vars: np.ndarray     # (5, n) the wiring the copy permutation comes from
    witness: list | None      # ints, or None: the case exists as tables only
    rows: list                # the rows whose gate it claims violated
    violation: list           # gate value per row of H
    copies_hold: bool
    kind: str                 # "single row", "low degree d", "copy only", "gate and copy", "blinder", "control"
    expect: int               # the oracle's rc: 0 or UNSAT
    blinders: list = field(default_factory=lambda: [0x51 + i for i in range(17)])
    deg_r: int | None = None  # degree of the violation polynomial as built (None: no gate is violated)
    good_vals: list = None    # a satisfying witness of the same circuit (the case before it was broken)

    @property
    def n(self) -> int:
        return 1 << self.log_n

    def tables(self):
        """(selectors (13, n, 4), wires (5, n, 4), pub (ni, 4), perm (5n,), k (5, 4), blinders (17, 4)), Montgomery."""
        sel = np.stack([synth.to_mont_array(c) for c in self.sel])
        wires = np.stack([synth.to_mont_array(c) for c in self.wires])
        return (sel, wires, synth.to_mont_array(self.pub).reshape(-1, 4), wiring_permutation(self.wire_vars), _k(),
                synth.to_mont_array(self.blinders))

    def witness_mont(self) -> np.ndarray:
        return synth.to_mont_array(self.witness)

    def good_witness_mont(self) -> np.ndarray:
        return synth.to_mont_array(self.good_vals)

    @property
    def good(self):
        """(wires, pub) ints of the satisfying witness: the control every refusal is followed by"""
        wv, v = self.wire_vars, self.good_vals
        return ([[v[int(x)] for x in wv[c]] for c in range(NW)], [v[int(wv[4, j])] for j in range(self.num_inputs)])


def _fresh(log_n, num_inputs, blank=(), seed=0):
    """The fresh-output circuit: (sel, wire_vars, values).  Variable 0 is zero, variable 1 + i is row i's output."""
    n = 1 << log_n
    rnd = random.Random(seed * 1000003 + log_n * 101 + num_inputs)
    sel = [[0] * n for _ in range(13)]
    wv = np.zeros((NW, n), dtype=np.uint32)
    vals = [0] + [0] * n
    for i in range(n):
        if i in blank:
            continue
        sel[synth.Q_O][i] = 1
        wv[4, i] = 1 + i
        if i < num_inputs:
            vals[1 + i] = rnd.randrange(R)
        else:
            sel[synth.Q_C][i] = rnd.randrange(R)
            vals[1 + i] = sel[synth.Q_C][i]
    return sel, wv, vals


def _case(name, log_n, num_inputs, sel, wv, vals, kind, rows, violation, copies_hold=True, table=None, pub=None,
          witness_ok=True, deg_r=None, expect=None, blinders=None, good_vals=None):
    n = 1 << log_n
    wires = table if table is not None else [[vals[int(wv[c, j])] for j in range(n)] for c in range(NW)]
    pub = pub if pub is not None else [vals[int(wv[4, j])] for j in range(num_inputs)]
    if expect is None:
        expect = UNSAT if (any(violation) or not copies_hold) else 0
    c = Case(name, log_n, num_inputs, sel, wires, pub, wv, list(vals) if witness_ok else None, rows, violation,
             copies_hold, kind, expect)
    if blinders is not None:
        c.blinders = blinders
    c.deg_r = deg_r
    c.good_vals = list(good_vals if good_vals is not None else vals)
    return c


def satisfied(log_n, num_inputs=3, seed=0) -> Case:
    """The fresh-output circuit with its satisfying witness."""
    sel, wv, vals = _fresh(log_n, num_inputs, seed=seed)
    return _case(f"satisfied_{log_n}", log_n, num_inputs, sel, wv, vals, "control", [], [0] * (1 << log_n))


# ---- one gate, one row ----------------------------------------------------------------------------------------------
def single_row(log_n: int, row: int, num_inputs: int = 3, delta: int = 1) -> Case:
    """w4 of one non-public row off by delta: that row's gate value is delta.  (A public row's input follows its w4 in
    a witness vector; `public_input` breaks those.)"""
    assert row >= num_inputs
    n = 1 << log_n
    sel, wv, vals = _fresh(log_n, num_inputs)
    good = list(vals)
    vals[1 + row] = (vals[1 + row] - delta) % R
    viol = [0] * n
    viol[row] = delta % R
    return _case(f"single_row_{log_n}_{row}", log_n, num_inputs, sel, wv, vals, "single row", [row], viol, deg_r=n - 1,
                 good_vals=good)


def single_rows(log_n: int, num_inputs: int = 3) -> list:
    """Row num_inputs, the last row, the scan's chunk edge CH - 1 / CH and a middle row."""
    n = 1 << log_n
    rows = sorted({num_inputs, n - 1, CH - 1, CH, n // 2 + 1} & set(range(num_inputs, n)))
    return [single_row(log_n, r, num_inputs) for r in rows]


# ---- public inputs (tables only) --------------------------------------------------------------------------------------
def public_input(log_n: int, which: int, num_inputs: int = 3) -> Case:
    """Public input `which` off by one while its row's w4 keeps its value: that row's gate value is 1."""
    n = 1 << log_n
    sel, wv, vals = _fresh(log_n, num_inputs)
    pub = [vals[1 + j] for j in range(num_inputs)]
    pub[which] = (pub[which] + 1) % R
    viol = [0] * n
    viol[which] = 1
    return _case(f"public_input_{log_n}_{which}", log_n, num_inputs, sel, wv, vals, "single row", [which], viol,
                 pub=pub, witness_ok=False, deg_r=n - 1)


def every_input_off(log_n: int, e: int = 1) -> Case:
    """witness_shapes.every_row_public with every public input off by e: the violation is the constant e."""
    from witness_shapes import every_row_public
    shp = every_row_public(log_n)
    n = 1 << log_n
    circ = shp.circ
    vals = [int.from_bytes(np.ascontiguousarray(circ.witness[v]).tobytes(), "little") * pow(2, -256, R) % R
            for v in range(circ.num_vars)]
    sel = [[0] * n for _ in range(13)]
    sel[synth.Q_O] = [1] * n
    wv = circ.wire_vars
    pub = [(vals[int(wv[4, j])] + e) % R for j in range(n)]
    return _case(f"every_input_off_{log_n}", log_n, n, sel, wv, vals, "low degree 0", list(range(n)), [e % R] * n,
                 pub=pub, witness_ok=False, deg_r=0)


# ---- copy constraints only ------------------------------------------------------------------------------------------
def copy_only(log_n: int, col: int, wrap: bool = False, num_inputs: int = 3) -> Case:
    """A shared variable on three positions the selectors ignore (w0..w3 of fresh-output rows, any wire of the blank
    last row); one of its positions in the table takes another value.  Every gate holds.  col: the column of the
    changed position (4: on the blank row).  wrap: the cycle runs through rows n - 1 and 0 and the change is on row
    n - 1, where z wraps around."""
    n = 1 << log_n
    sel, wv, vals = _fresh(log_n, num_inputs, blank=(n - 1,))
    u = len(vals)
    vals.append(random.Random(log_n * 7 + col).randrange(1, R))
    if wrap:
        where = [(col, n - 1), ((col + 1) % 4, 0), ((col + 2) % 4, n // 2)]
    elif col == 4:
        where = [(4, n - 1), (0, 5 % n), (3, 9 % n)]
    else:
        where = [(col, n // 2 - 1), ((col + 1) % 4, 2), ((col + 3) % 4, n - 3)]
    for c, j in where:
        wv[c, j] = u
    table = [[vals[int(wv[c, j])] for j in range(n)] for c in range(NW)]
    c0, j0 = where[0]
    table[c0][j0] = (table[c0][j0] + 1) % R
    return _case(f"copy_only_{log_n}_{col}{'_wrap' if wrap else ''}", log_n, num_inputs, sel, wv, vals, "copy only", [],
                 [0] * n, copies_hold=False, table=table, witness_ok=False)


def gate_and_copy(log_n: int, num_inputs: int = 3) -> Case:
    """copy_only(col 0) and a single-row gate violation in the same table."""
    c = copy_only(log_n, 0, num_inputs=num_inputs)
    n = 1 << log_n
    row = n // 2 + 1
    c.wires[4][row] = (c.wires[4][row] - 1) % R
    c.violation = [0] * n
    c.violation[row] = 1
    c.rows, c.kind, c.name, c.deg_r = [row], "gate and copy", f"gate_and_copy_{log_n}", n - 1
    return c


# ---- low-degree violations ------------------------------------------------------------------------------------------
LOW_DEGREE = ["const", "x", "roots7", "roots8"]


def low_degree(log_n: int, p: str) -> Case:
    """Fresh-output circuit, w4 on every row i shifted by -p(w^i): p = 1, p = X, or p = prod_{t in S} (X - w^t) with S
    the |S| public rows (7 or 8), so that the shift touches no public row.  deg p <= 7 is missed by six cosets."""
    n = 1 << log_n
    w = omega(log_n)
    if p in ("const", "x"):
        ni, roots = 0, []
    else:
        ni = int(p[len("roots"):])
        roots = [pow(w, t, R) for t in range(ni)]
    assert ni < n
    sel, wv, vals = _fresh(log_n, ni)
    good = list(vals)
    viol, x = [], 1
    for i in range(n):
        if p == "const":
            v = 1
        elif p == "x":
            v = x
        else:
            v = 1
            for rt in roots:
                v = v * (x - rt) % R
        viol.append(v)
        vals[1 + i] = (vals[1 + i] - v) % R
        x = x * w % R
    deg = {"const": 0, "x": 1}.get(p, ni)
    return _case(f"low_degree_{log_n}_{p}", log_n, ni, sel, wv, vals, f"low degree {deg}",
                 [i for i in range(n) if viol[i]], viol, deg_r=deg, good_vals=good)


def low_degree_sizes(p: str) -> list:
    """2^2 and 2^3 (eight cosets, a control) take p = 1 and X; the |S| = 7 and 8 products need n > |S|."""
    sizes = [2, 3, 4, 5, 10, 16] if p in ("const", "x") else [4, 5, 10, 16]
    return sizes


# ---- blinders ------------------------------------------------------------------------------------------------------
# a zero at 2i + 1 (each wire's X^(n+1) blinder) or 12 (z's X^(n+2) blinder) zeroes the quotient's coefficient 5n + 7,
# which round 3's bit 1 refuses, as the reference's degree check does
BLINDERS_TOP = [1, 3, 5, 7, 9, 12]


def blinder_zero(log_n: int, index: int, num_inputs: int = 3) -> Case:
    c = satisfied(log_n, num_inputs)
    bl = list(c.blinders)
    bl[index] = 0
    c.blinders = bl
    c.kind, c.name = "blinder", f"blinder_zero_{log_n}_{index}"
    c.expect = UNSAT if index in BLINDERS_TOP else 0
    return c


def catalogue(max_log_n: int = 10) -> list:
    """Every case up to domain 2^max_log_n."""
    out = []
    for log_n in (4, 5):
        out += single_rows(log_n)
        out += [public_input(log_n, 0), public_input(log_n, 2)]
        out += [copy_only(log_n, col) for col in range(NW)] + [copy_only(log_n, 1, wrap=True)]
        out.append(gate_and_copy(log_n))
    for p in LOW_DEGREE:
        out += [low_degree(s, p) for s in low_degree_sizes(p) if s <= max_log_n]
    out += [every_input_off(s) for s in (5, 10) if s <= max_log_n]
    out += [blinder_zero(4, i) for i in range(17)]
    return out
