"""Synthetic TurboPlonk circuits for benchmarks and parity tests.

The reference's circuits are synthesised by Rust code (crates/circuits/circuits-core) that cannot
run here, so the benchmark of the VALID-MATCH-class statement
(`IntentAndBalancePrivateSettlementCircuit`, SURVEY.md §0.1) uses a synthetic circuit of the same
shape: 5 wire columns, the 13 TurboPlonk selector columns
q_lc[4] q_mul[2] q_hash[4] q_o q_c q_ecc, public-input gates first, a gate mix dominated by
Poseidon2-style x^5 gates (one permutation = 195 such gates, SURVEY.md §2.1), dense copy
constraints, zero-padding to the domain size.  Everything here is host-side input generation
(Python integers); none of it is on the proving path.
"""
from __future__ import annotations

import random
from dataclasses import dataclass

import numpy as np

R = 0x30644E72E131A029B85045B68181585D2833E84879B97091_43E1F593F0000001
N_WIRES = 5
N_SELECTORS = 13
# selector column order (mpc-jellyfish TurboPlonk, as used by
# circuits-core/src/zk_gadgets/primitives/poseidon/gates.rs:78-100)
Q_LC, Q_MUL, Q_HASH, Q_O, Q_C, Q_ECC = 0, 4, 6, 10, 11, 12


def to_mont_array(vals) -> np.ndarray:
    """list of ints (< r) -> (len, 4) uint64 Montgomery limbs (little-endian, the ABI's layout)."""
    vals = list(vals)
    if not vals:
        return np.zeros((0, 4), dtype=np.uint64)
    zero = bytes(32)
    buf = b"".join(((v << 256) % R).to_bytes(32, "little") if v else zero for v in vals)
    return np.frombuffer(buf, dtype="<u8").reshape(len(vals), 4).astype(np.uint64, copy=True)


@dataclass
class SynthCircuit:
    log_n: int
    num_inputs: int
    k: np.ndarray            # (5, 4) coset representatives, Montgomery
    selectors: np.ndarray    # (13, n, 4) selector evaluations over H, Montgomery
    perm: np.ndarray         # (5n,) uint64: perm[i*n + j] = i'*n + j'
    wires: np.ndarray        # (5, n, 4) wire values, Montgomery
    pub_inputs: np.ndarray   # (num_inputs, 4) Montgomery
    n_gates: int             # gates before padding
    # integer views for checks
    selectors_int: list
    wires_int: list
    pub_inputs_int: list
    # fingerprint of the witness-independent part (gate placement, wiring, selector values), comparable within one
    # process; 0 = not computed.  A constraint system may also be finalized `wires_only` (selectors / perm left None)
    # when the caller only needs the per-proof tables: the key already holds the structure.
    structure_digest: int = 0
    # the circuit as wiring + witness vector (b200_plonk_preprocess_wiring / b200_plonk_prove_witness):
    # wires[i, j] = witness[wire_vars[i, j]].  A constraint system may be finalized `witness_only` (wires left None too).
    wire_vars: np.ndarray = None   # (5, n) uint32: the variable on wire i of row j
    witness: np.ndarray = None     # (num_vars, 4) Montgomery

    @property
    def num_vars(self) -> int:
        return 0 if self.witness is None else len(self.witness)

    @property
    def n(self) -> int:
        return 1 << self.log_n


def gate_value(q, w, pi):
    """Left-hand side of the TurboPlonk gate equation (must be 0 mod r)."""
    acc = q[Q_C] + pi
    for j in range(4):
        acc += q[Q_LC + j] * w[j] + q[Q_HASH + j] * pow(w[j], 5, R)
    acc += q[Q_MUL] * w[0] * w[1] + q[Q_MUL + 1] * w[2] * w[3]
    acc += q[Q_ECC] * w[0] * w[1] * w[2] * w[3] * w[4]
    acc -= q[Q_O] * w[4]
    return acc % R


def synth_circuit(log_n: int, num_inputs: int = 17, seed: int = 0xB200, fill: float = 0.93,
                  check: bool = False, link=None) -> SynthCircuit:
    """link = (alignment, offset, values): a proof-linking group.  Value i is pinned to wire 0 of
    row (offset + i) * n / 2^alignment — the row whose domain element is the (offset + i)-th
    2^alignment-th root of unity — with all selectors zero, as mpc-relation places link gates
    (SURVEY.md App. A, round 1); later gates may reuse the value through copy constraints."""
    n = 1 << log_n
    link_rows = {}
    if link is not None:
        alignment, offset, link_vals = link
        assert alignment <= log_n
        for i, v in enumerate(link_vals):
            link_rows[(offset + i) << (log_n - alignment)] = v % R
        assert min(link_rows) >= num_inputs, "link group collides with the public-input rows"
    rnd = random.Random(seed)
    n_gates = max(num_inputs + 1, min(n - 1, int(n * fill)))
    values = [0]                       # variable 0 is the constant zero
    positions = [[]]                   # per variable: (wire, row) occurrences
    sel = [[0] * n for _ in range(N_SELECTORS)]
    wire_var = [[0] * n for _ in range(N_WIRES)]
    pub_inputs = []

    def new_var(v):
        values.append(v % R)
        positions.append([])
        return len(values) - 1

    def pick():
        # recent variables are reused more often, like the rounds of a hash permutation
        hi = len(values) - 1
        if hi == 0:
            return 0
        if rnd.random() < 0.8:
            return max(0, hi - rnd.randrange(min(hi + 1, 12)))
        return rnd.randrange(hi + 1)

    for row in range(n_gates):
        q = [0] * N_SELECTORS
        if row in link_rows:           # link gate: wire 0 carries the shared value, no constraint
            var = new_var(link_rows[row])
            for wcol, vv in enumerate([var, 0, 0, 0, 0]):
                wire_var[wcol][row] = vv
                positions[vv].append((wcol, row))
            continue
        if row < num_inputs:           # IO gate: w4 = public input
            pi = rnd.randrange(R)
            pub_inputs.append(pi)
            ins = [0, 0, 0, 0]
            q[Q_O] = 1
            out = new_var(pi)
        else:
            ins = [pick() for _ in range(4)]
            wv = [values[v] for v in ins]
            kind = rnd.random()
            q[Q_O] = 1
            q[Q_C] = rnd.randrange(R)
            if kind < 0.80:            # Poseidon2-style power-5 gate
                for j in range(4):
                    q[Q_HASH + j] = rnd.randrange(R)
                res = q[Q_C] + sum(q[Q_HASH + j] * pow(wv[j], 5, R) for j in range(4))
            elif kind < 0.90:          # linear combination
                for j in range(4):
                    q[Q_LC + j] = rnd.randrange(R)
                res = q[Q_C] + sum(q[Q_LC + j] * wv[j] for j in range(4))
            elif kind < 0.98:          # two multiplications
                q[Q_MUL], q[Q_MUL + 1] = rnd.randrange(R), rnd.randrange(R)
                res = q[Q_C] + q[Q_MUL] * wv[0] * wv[1] + q[Q_MUL + 1] * wv[2] * wv[3]
            else:                      # ecc-style gate: the product term contains w4 itself
                q[Q_ECC] = rnd.randrange(R)
                q[Q_LC] = rnd.randrange(R)
                prod = wv[0] * wv[1] * wv[2] * wv[3] % R
                denom = (q[Q_O] - q[Q_ECC] * prod) % R
                if denom == 0:
                    q[Q_ECC] = 0
                    denom = q[Q_O]
                res = (q[Q_C] + q[Q_LC] * wv[0]) * pow(denom, -1, R)
            out = new_var(res)
        for s in range(N_SELECTORS):
            sel[s][row] = q[s]
        cols = ins + [out]
        for wcol, var in enumerate(cols):
            wire_var[wcol][row] = var
            positions[var].append((wcol, row))
    # padding rows: all selectors zero, all wires the zero variable
    for row in range(n_gates, n):
        cols = [0] * N_WIRES
        if row in link_rows:
            cols[0] = new_var(link_rows[row])
        for wcol in range(N_WIRES):
            wire_var[wcol][row] = cols[wcol]
            positions[cols[wcol]].append((wcol, row))

    # copy-constraint permutation: each variable's occurrences form one cycle
    perm = np.empty(N_WIRES * n, dtype=np.uint64)
    for occ in positions:
        for a, b in zip(occ, occ[1:] + occ[:1]):
            perm[a[0] * n + a[1]] = b[0] * n + b[1]

    wires_int = [[values[wire_var[w][row]] for row in range(n)] for w in range(N_WIRES)]
    if check:
        for row in range(n):
            pi = pub_inputs[row] if row < num_inputs else 0
            assert gate_value([sel[s][row] for s in range(N_SELECTORS)], [wires_int[w][row] for w in range(N_WIRES)], pi) == 0, row

    k_int = [pow(5, i, R) for i in range(N_WIRES)]  # disjoint cosets k_i * H (5 generates Fr*)
    return SynthCircuit(
        log_n=log_n, num_inputs=num_inputs, k=to_mont_array(k_int),
        selectors=np.stack([to_mont_array(col) for col in sel]), perm=perm,
        wires=np.stack([to_mont_array(col) for col in wires_int]),
        pub_inputs=to_mont_array(pub_inputs), n_gates=n_gates,
        selectors_int=sel, wires_int=wires_int, pub_inputs_int=pub_inputs,
        wire_vars=np.array(wire_var, dtype=np.uint32), witness=to_mont_array(values))


def splitmix_blinders(seed: int, count: int = 17) -> np.ndarray:
    """Deterministic stand-in for the 17 field elements the reference draws from thread_rng()
    (traits.rs:994): SplitMix64 words reduced mod r, Montgomery form."""
    mask = (1 << 64) - 1
    s = seed & mask
    vals = []
    for _ in range(count):
        v = 0
        for kk in range(4):
            s = (s + 0x9E3779B97F4A7C15) & mask
            z = s
            z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & mask
            z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & mask
            v |= (z ^ (z >> 31)) << (64 * kk)
        vals.append(v % R)
    return to_mont_array(vals)
