"""Test infrastructure: circuits given as wiring + witness vector at the shapes where deriving the copy permutation on
the device (`renegade_b200/csrc/wiring.cu`) and gathering the wire tables (`k_gather_wires`) can go wrong.

`wiring_permutation` sorts the keys `variable << 32 | position` by their bits [0, end_bit): the 32 position bits and
as many bits of the variable index as num_vars - 1 has, at least one (`END_BIT_MIN` = 33 is read from wiring.cu, as
`msm_digits.py` reads msm.cu).  `k_wiring_cycles` then links each group of equal variables, one thread per sorted key
in blocks of `CYCLE_THREADS`, finding a group's head by binary search.

A single proof stages a host witness in the context's NTT scratch, which `preprocess` has already sized to NS * m
elements (m = cosets * n) and `prove()` to 7m per proof; only a witness longer than both grows it.  NS, the coset
rule and the 7 are read from plonk.cu (`staging_floor`).

Each builder returns a `Shape`: the circuit (a `synth.SynthCircuit`), its num_vars, and the claim the shape is built
for, which tests/test_witness_shapes_cpu.py checks.  A shape whose num_vars is too large for a witness vector in memory
(2^31 + 1, 2^32 - 1) carries its used variables' values in `values` and no witness: its key can be made, it cannot be
proved."""
from __future__ import annotations

import dataclasses
import os
import random
import re
from dataclasses import dataclass, field

import numpy as np

from renegade_b200 import synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
R = synth.R
NW = synth.N_WIRES


def _source(name: str) -> str:
    with open(os.path.join(ROOT, "renegade_b200", "csrc", name)) as f:
        return f.read()


def _constants(name: str, pattern: str) -> tuple:
    m = re.search(pattern, _source(name))
    assert m, f"{name} no longer matches {pattern!r}"
    return tuple(int(g) for g in m.groups())


END_BIT_MIN, = _constants("wiring.cu", r"int end_bit = (\d+);")
CYCLE_THREADS, = _constants("wiring.cu", r"B200_LAUNCH\(k_wiring_cycles, grid, (\d+),")
NS, = _constants("plonk.cu", r"constexpr int NS = (\d+);")
# nc = log_n >= COSET_SWITCH ? COSETS_LARGE : COSETS_SMALL
COSET_SWITCH, COSETS_LARGE, COSETS_SMALL = _constants("plonk.cu", r"const int nc = log_n >= (\d+) \? (\d+) : (\d+);")
STAGE_PER_M, = _constants("plonk.cu", r"std::max\((\d+) \* m, from_witness \? pk->num_vars : 0\)")
assert re.search(r"ntt_scratch\.reserve\(\(size_t\)NS \* m \* sizeof\(fe\)\)", _source("plonk.cu")), \
    "preprocess no longer reserves NS * m elements of NTT scratch"
MAX_WITNESS_VARS = (1 << 24) + 1  # the largest witness vector a shape materialises (512 MiB)


def end_bit(num_vars: int) -> int:
    """wiring.cu's sort width: the position's 32 bits and as many bits of the index as num_vars - 1 has."""
    b = END_BIT_MIN
    while b < 64 and (num_vars - 1) >> (b - 32):
        b += 1
    return b


def index_bits(num_vars: int) -> int:
    """Bits of the variable index the sort reads (end_bit - 32)."""
    return end_bit(num_vars) - 32


def staging_floor(log_n: int) -> int:
    """Elements of NTT scratch a context holds once it has preprocessed and proved a key of domain 2^log_n: NS * m from
    preprocess, STAGE_PER_M * m from a proof (m = cosets * n).  A witness vector longer than this grows the scratch."""
    m = (COSETS_LARGE if log_n >= COSET_SWITCH else COSETS_SMALL) << log_n
    return max(NS, STAGE_PER_M) * m


@dataclass
class Shape:
    name: str
    circ: synth.SynthCircuit  # circ.witness is None when num_vars > MAX_WITNESS_VARS
    num_vars: int
    claim: str
    values: dict = field(default_factory=dict)  # used variable -> value (int), for the shapes without a witness
    top_pairs: list = field(default_factory=list)  # (v, v + 2^(b-1)) pairs interleaved position by position


def _k():
    return synth.to_mont_array([pow(5, i, R) for i in range(NW)])


def _finish(log_n, num_inputs, selectors, wire_vars, witness, n_gates=None) -> synth.SynthCircuit:
    """A SynthCircuit with the derived fields filled in: the expanded table and the public inputs.  perm is left None:
    the tests take the permutation from test_prove_witness_cpu.wiring_permutation."""
    wv = np.ascontiguousarray(wire_vars, dtype=np.uint32).reshape(NW, 1 << log_n)
    wires = witness[wv] if witness is not None else None
    pub = witness[wv[4, :num_inputs]] if witness is not None else None
    return synth.SynthCircuit(log_n=log_n, num_inputs=num_inputs, k=_k(), selectors=selectors, perm=None, wires=wires,
                              pub_inputs=pub, n_gates=n_gates if n_gates is not None else 1 << log_n,
                              selectors_int=None, wires_int=None, pub_inputs_int=None, wire_vars=wv, witness=witness)


def sparse_witness(num_vars: int, values: dict) -> np.ndarray:
    """(num_vars, 4) Montgomery witness: the given variables set, every other one zero (np.zeros pages lazily)."""
    w = np.zeros((num_vars, 4), dtype=np.uint64)
    keys = sorted(values)
    w[np.array(keys, dtype=np.int64)] = synth.to_mont_array([values[v] for v in keys])
    return w


# ---- index width --------------------------------------------------------------------------------------------------
# num_vars either side of the sort's digit boundaries and at the top of a 32-bit index
INDEX_WIDTHS = [1, 2, 256, 257, 1 << 16, (1 << 16) + 1, 1 << 24, (1 << 24) + 1, (1 << 31) + 1, (1 << 32) - 1]


def index_width(num_vars: int, log_n: int = 4, seed: int = 0) -> Shape:
    """No gate constraints; the wiring uses 0 and num_vars - 1, and pairs v, v + 2^(b-1) (b = the index bits the sort
    reads, so the pair differs only in the top one) are interleaved position by position: a sort one bit short would
    merge each pair into one cycle."""
    n = 1 << log_n
    rnd = random.Random(seed ^ num_vars)
    b = (num_vars - 1).bit_length()
    pairs = []
    if b:
        h = 1 << (b - 1)
        for v in (0, h - 1, num_vars - 1 - h):
            if v + h < num_vars and (v, v + h) not in pairs:
                pairs.append((v, v + h))
    order = [v for p in pairs for v in p] or [0]
    wv = np.array([order[p % len(order)] for p in range(NW * n)], dtype=np.uint32)
    used = sorted(set(order))
    values = {v: rnd.randrange(R) for v in used}
    witness = sparse_witness(num_vars, values) if num_vars <= MAX_WITNESS_VARS else None
    circ = _finish(log_n, 0, np.zeros((13, n, 4), dtype=np.uint64), wv, witness)
    return Shape(f"index_width_{num_vars}", circ, num_vars,
                 f"end_bit {end_bit(num_vars)}; indices 0 and {num_vars - 1} used; top-bit pairs {pairs}",
                 values=values, top_pairs=pairs)


# ---- cycle shapes (the service's sizes: 2^16, 2^17) ----------------------------------------------------------------
def _random_values(count, rnd):
    return synth.to_mont_array([rnd.randrange(R) for _ in range(count)])


def one_variable(log_n: int) -> Shape:
    """One variable on all 5n positions: one cycle through the whole table."""
    n = 1 << log_n
    circ = _finish(log_n, 0, np.zeros((13, n, 4), dtype=np.uint64), np.zeros(NW * n, dtype=np.uint32),
                   _random_values(1, random.Random(log_n)))
    return Shape(f"one_variable_{log_n}", circ, 1, f"one cycle of {NW * n} positions")


def each_once_descending(log_n: int) -> Shape:
    """Every position its own variable, numbered in descending position order: 5n fixed points."""
    n = 1 << log_n
    wv = np.arange(NW * n, dtype=np.uint32)[::-1].copy()
    circ = _finish(log_n, 0, np.zeros((13, n, 4), dtype=np.uint64), wv, _random_values(NW * n, random.Random(log_n + 1)))
    return Shape(f"each_once_{log_n}", circ, NW * n, f"{NW * n} cycles of length 1")


def block_boundary_pairs(log_n: int, seed: int = 7) -> Shape:
    """In sorted order (variable, then position) the variables take 1, 2, 2, 2, ... positions, so a variable of exactly
    two positions sits on sorted indices t - 1 and t of every thread-block boundary t of k_wiring_cycles (the second
    of them finds its head by binary search into the previous block).  The positions themselves are shuffled."""
    n = 1 << log_n
    total = NW * n
    pos = np.random.default_rng(seed).permutation(total)
    var_of_sorted = (np.arange(total) + 1) // 2        # sizes 1, 2, 2, ...
    wv = np.empty(total, dtype=np.uint32)
    wv[pos] = var_of_sorted
    nv = int(var_of_sorted[-1]) + 1
    circ = _finish(log_n, 0, np.zeros((13, n, 4), dtype=np.uint64), wv, _random_values(nv, random.Random(seed)))
    return Shape(f"block_boundary_{log_n}", circ, nv,
                 f"a two-position variable on sorted indices t - 1, t of each multiple t of {CYCLE_THREADS}")


def stride_n(log_n: int) -> Shape:
    """Variable j on row j of every wire column: n cycles of 5 positions, n apart."""
    n = 1 << log_n
    wv = np.tile(np.arange(n, dtype=np.uint32), NW)
    circ = _finish(log_n, 0, np.zeros((13, n, 4), dtype=np.uint64), wv, _random_values(n, random.Random(log_n + 2)))
    return Shape(f"stride_n_{log_n}", circ, n, f"{n} cycles (j, n + j, ..., 4n + j)")


def dense(log_n: int, num_inputs: int = None, seed: int = 0xB200) -> Shape:
    """The synthetic gate mix (synth.synth_circuit): hash, linear, product and ecc gates, dense copy constraints.
    num_inputs: 17 public inputs (bench.py's), fewer where the domain is small."""
    if num_inputs is None:
        num_inputs = min(17, (1 << log_n) // 2)
    circ = synth.synth_circuit(log_n, num_inputs=num_inputs, seed=seed)
    return Shape(f"dense_{log_n}", circ, circ.num_vars, "satisfied gate mix")


# ---- public inputs -----------------------------------------------------------------------------------------------
def public_inputs(log_n: int, num_inputs: int, shared: bool = False, zero: bool = False, seed: int = 21) -> Shape:
    """The synthetic gate mix with `num_inputs` public-input rows (1 <= num_inputs < n, or 0).  shared: the variable of
    row 1 is public on row num_inputs - 1 too; zero: the constant-zero variable (0) is the public input of row 0."""
    n = 1 << log_n
    circ = synth.synth_circuit(log_n, num_inputs=num_inputs, seed=seed + log_n)
    wv = circ.wire_vars.copy()
    if shared:
        assert num_inputs >= 3
        wv[4, num_inputs - 1] = wv[4, 1]
    if zero:
        assert num_inputs >= 1 and not circ.witness[0].any()
        wv[4, 0] = 0
    out = _finish(log_n, num_inputs, circ.selectors, wv, circ.witness, circ.n_gates)
    return Shape(f"public_inputs_{log_n}_{num_inputs}{'_shared' if shared else ''}{'_zero' if zero else ''}", out,
                 circ.num_vars, f"{num_inputs} of {n} rows public" + (", one variable on two" if shared else "")
                 + (", the zero variable public" if zero else ""))


def every_row_public(log_n: int, seed: int = 5) -> Shape:
    """num_inputs = n: every row is a public-input gate (q_o = 1, w4 = its public variable), the other wires random
    earlier variables.  Row 0's public variable is the constant zero, row n - 1 repeats row 1's."""
    n = 1 << log_n
    rnd = random.Random(seed + log_n)
    values = [0]
    wv = np.zeros((NW, n), dtype=np.uint32)
    for j in range(n):
        if j == 0:
            out = 0
        elif j == n - 1:
            out = int(wv[4, 1])
        else:
            values.append(rnd.randrange(R))
            out = len(values) - 1
        wv[4, j] = out
        for i in range(4):
            wv[i, j] = rnd.randrange(len(values))
    sel = np.zeros((13, n, 4), dtype=np.uint64)
    sel[synth.Q_O] = synth.to_mont_array([1])[0]
    circ = _finish(log_n, n, sel, wv, synth.to_mont_array(values))
    return Shape(f"every_row_public_{log_n}", circ, len(values),
                 f"all {n} rows public, the zero variable on row 0, one variable on rows 1 and {n - 1}")


# ---- unused variables ----------------------------------------------------------------------------------------------
def unused_variables(log_n: int, factor: int = 128, num_inputs: int = 3, seed: int = 31) -> Shape:
    """The synthetic gate mix with its variables relabelled into [0, factor * n), the highest index used.  With the
    default factor the witness vector is longer than `staging_floor` (at most 104n), so staging it grows the NTT
    scratch of a context that holds only keys of this domain size."""
    n = 1 << log_n
    circ = synth.synth_circuit(log_n, num_inputs=num_inputs, seed=seed + log_n)
    nv = factor * n
    rng = np.random.default_rng(seed)
    used = circ.num_vars
    label = np.sort(rng.choice(nv - 1, size=used - 1, replace=False)) if used > 1 else np.zeros(0, dtype=np.int64)
    label = np.r_[label, nv - 1] if used > 1 else np.array([nv - 1])
    label = rng.permutation(label)                      # variable v -> label[v]
    witness = synth.to_mont_array([random.Random(seed).randrange(R) for _ in range(nv)])
    witness[label] = circ.witness
    wv = label[circ.wire_vars].astype(np.uint32)
    out = _finish(log_n, num_inputs, circ.selectors, wv, witness, circ.n_gates)
    return Shape(f"unused_variables_{log_n}", out, nv, f"{used} of {nv} variables used, the last one among them")


# ---- distinct witnesses of one circuit ---------------------------------------------------------------------------------
def dense_witnesses(circ: synth.SynthCircuit, count: int, seed: int = 0) -> list:
    """`count` witness vectors of a synth.synth_circuit circuit (no link group), each with fresh public inputs and
    every other variable recomputed from the gate that outputs it: w4 = (q_c + sum q_lc w + sum q_hash w^5 + q_mul0 w0 w1
    + q_mul1 w2 w3) / (q_o - q_ecc w0 w1 w2 w3).  Each satisfies the circuit; no two are equal."""
    rnd = random.Random(seed)
    wv, sel = circ.wire_vars, circ.selectors_int
    out = []
    for _ in range(count):
        val = [0] * circ.num_vars  # variable 0 stays the constant zero
        for j in range(circ.n_gates):
            v = int(wv[4, j])
            if j < circ.num_inputs:
                val[v] = rnd.randrange(R)
                continue
            w = [val[int(wv[i, j])] for i in range(4)]
            q = [sel[s][j] for s in range(synth.N_SELECTORS)]
            num = q[synth.Q_C] + q[synth.Q_MUL] * w[0] * w[1] + q[synth.Q_MUL + 1] * w[2] * w[3]
            num += sum(q[synth.Q_LC + i] * w[i] + q[synth.Q_HASH + i] * pow(w[i], 5, R) for i in range(4))
            den = (q[synth.Q_O] - q[synth.Q_ECC] * w[0] * w[1] * w[2] * w[3]) % R
            assert den, (j, "the output of this gate is not determined by its inputs")
            val[v] = num * pow(den, -1, R) % R
        out.append(synth.to_mont_array(val))
    return out


def with_witness(circ: synth.SynthCircuit, witness: np.ndarray) -> synth.SynthCircuit:
    """The same circuit with another witness vector (and its table and public inputs)."""
    return dataclasses.replace(circ, witness=witness, wires=witness[circ.wire_vars],
                               pub_inputs=witness[circ.wire_vars[4, :circ.num_inputs]], wires_int=None, pub_inputs_int=None)
