"""Host-side constraint system: the caller side of the proving boundary.

The reference synthesises its circuits in Rust (`SingleProverCircuit::prove`, circuit-types/src/traits.rs:976-991:
create the witness variables, `apply_constraints`, `finalize_for_arithmetization`) on mpc-relation's
`PlonkCircuit<ScalarField>` and hands the finished tables to the prover.  That code cannot run here (no cargo), so this
module restates the part of that interface the proving path consumes — variables, the TurboPlonk gate set with its 13
selector columns, copy constraints, public-input gates first, zero padding to the domain — and the reference's own
Poseidon2 and Merkle gadgets on top of it, so that tests and benches can prove circuits with the reference's gate
structure instead of random tables:

  * `PlonkCircuit`               mpc-relation `PlonkCircuit` (as used through `mpc_relation::traits::Circuit`)
  * `FusedExternalSboxMDSGate`,
    `FusedInternalSboxMDSGate`   circuits-core/src/zk_gadgets/primitives/poseidon/gates.rs:27-100, 117-179
  * `PoseidonHashGadget`         .../poseidon/hash.rs:56-423 (195 gates per permutation)
  * `PoseidonMerkleHashGadget`   .../primitives/merkle.rs:13-126
  * `ToBitsGadget`, `BitRangeGadget`                       .../primitives/bits.rs:22-110
  * `EqZeroGadget`, `GreaterThanEq(Zero)Gadget`            .../primitives/comparators.rs:17-260
  * `CSPRNGGadget`, `StreamCipherGadget`, `RecoveryIdGadget`,
    `CommitmentGadget`, `AmountGadget`                     .../state_primitives/{csprng,stream_cipher,recovery_id,
                                                           commitment}.rs, primitives/bitlength.rs
  * `PoseidonCSPRNG`, `StateWrapper`                       darkpool-types/src/{csprng,state_wrapper}.rs (native side)
  * `Poseidon2Sponge`,
    `compute_poseidon_hash`      crates/crypto/src/hash/poseidon2.rs:25-209, hash/mod.rs:12-18 (native, for witnesses)

Everything here is host-side input generation on Python integers; the tables `finalize_for_arithmetization` returns are
exactly what `b200_plonk_preprocess` / `b200_plonk_prove` take (same layout as renegade_b200/synth.py).
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import List, Sequence

import numpy as np

from renegade_b200.poseidon2_constants import CAPACITY, FULL_ROUND_CONSTANTS, PARTIAL_ROUND_CONSTANTS, R_F, R_P, RATE
from renegade_b200.synth import N_SELECTORS, N_WIRES, Q_C, Q_ECC, Q_HASH, Q_LC, Q_MUL, Q_O, R, SynthCircuit, gate_value, to_mont_array

GATE_WIDTH = 4
Variable = int


class CircuitError(Exception):
    """mpc-relation `CircuitError` (surfaces as `ProverError::Circuit`, circuit-types/src/errors.rs:33-58)."""


# ---------------------------------------------------------------------------------------------
# Gates: one row of the 13 selector columns
# ---------------------------------------------------------------------------------------------
@dataclass
class Gate:
    """mpc-relation `Gate`: q_lc[4], q_mul[2], q_hash[4], q_o, q_c, q_ecc (all zero by default).
    Equation: q_c + PI + sum q_lc w + q_mul0 w0 w1 + q_mul1 w2 w3 + sum q_hash w^5 + q_ecc w0 w1 w2 w3 w4 = q_o w4."""
    name: str = "Gate"
    q_lc: Sequence[int] = (0, 0, 0, 0)
    q_mul: Sequence[int] = (0, 0)
    q_hash: Sequence[int] = (0, 0, 0, 0)
    q_o: int = 0
    q_c: int = 0
    q_ecc: int = 0

    def selectors(self) -> List[int]:
        q = [0] * N_SELECTORS
        for j in range(4):
            q[Q_LC + j] = self.q_lc[j] % R
            q[Q_HASH + j] = self.q_hash[j] % R
        q[Q_MUL], q[Q_MUL + 1] = self.q_mul[0] % R, self.q_mul[1] % R
        q[Q_O], q[Q_C], q[Q_ECC] = self.q_o % R, self.q_c % R, self.q_ecc % R
        return q


def PaddingGate() -> Gate:
    return Gate("PaddingGate")


def IoGate() -> Gate:
    """w4 = public input (the public-input polynomial supplies the value)."""
    return Gate("IoGate", q_o=1)


def ConstantGate(c: int) -> Gate:
    return Gate("ConstantGate", q_c=c, q_o=1)


def AdditionGate() -> Gate:
    return Gate("AdditionGate", q_lc=(1, 1, 0, 0), q_o=1)


def SubtractionGate() -> Gate:
    return Gate("SubtractionGate", q_lc=(1, -1, 0, 0), q_o=1)


def MultiplicationGate() -> Gate:
    return Gate("MultiplicationGate", q_mul=(1, 0), q_o=1)


def LinCombGate(coeffs: Sequence[int]) -> Gate:
    return Gate("LinCombGate", q_lc=tuple(coeffs), q_o=1)


def EqualityGate() -> Gate:
    return Gate("EqualityGate", q_lc=(1, -1, 0, 0))


def BoolGate() -> Gate:
    """wires (a, a, 0, 0, a): a * a = a."""
    return Gate("BoolGate", q_mul=(1, 0), q_o=1)


def MulAddGate(q_mul: Sequence[int]) -> Gate:
    """wires (a, b, c, d, out): q0 * a * b + q1 * c * d = out."""
    return Gate("MulAddGate", q_mul=tuple(q_mul), q_o=1)


def ConstantAdditionGate(c: int) -> Gate:
    return Gate("ConstantAdditionGate", q_lc=(1, 0, 0, 0), q_c=c, q_o=1)


def MuxGate() -> Gate:
    """wires (sel, a, sel, b, out): out = sel * a - sel * b + b = if sel { a } else { b }."""
    return Gate("MuxGate", q_lc=(0, 0, 0, 1), q_mul=(1, -1), q_o=1)


def pow5(x: int) -> int:
    return pow(x, 5, R)


class FusedExternalSboxMDSGate(Gate):
    """poseidon/gates.rs:27-100: wires (state_curr, s0, s1, s2, out); out = rc + sum f(w), f = x^5 if `apply_sbox`
    else x — the external MDS circ(2, 1, 1) row of element `state_curr` (each element plus the sum of all three)
    fused with the next round's constant."""

    def __init__(self, apply_sbox: bool, round_constant: int):
        ones, zeros = (1, 1, 1, 1), (0, 0, 0, 0)
        super().__init__("FusedExternalSboxMDSGate", q_lc=zeros if apply_sbox else ones,
                         q_hash=ones if apply_sbox else zeros, q_o=1, q_c=round_constant)
        self.apply_sbox = apply_sbox

    def compute_output(self, state_curr: int, s0: int, s1: int, s2: int) -> int:
        el = [state_curr, s0, s1, s2]
        if self.apply_sbox:
            el = [pow5(x) for x in el]
        return (self.q_c + sum(el)) % R


class FusedInternalSboxMDSGate(Gate):
    """poseidon/gates.rs:117-179: out = rc + coeff * g(state_curr) + s0^5 + s1 + s2, g = x^5 if `apply_sbox` else x —
    a row of the internal matrix [[2,1,1],[1,2,1],[1,1,3]] applied to (s0^5, s1, s2), fused with the next constant."""

    def __init__(self, apply_sbox: bool, next_round_constant: int, state_elem_coeff: int):
        c = state_elem_coeff
        super().__init__("FusedInternalSboxMDSGate",
                         q_hash=(c, 1, 0, 0) if apply_sbox else (0, 1, 0, 0),
                         q_lc=(0, 0, 1, 1) if apply_sbox else (c, 0, 1, 1), q_o=1, q_c=next_round_constant)
        self.apply_sbox, self.coeff = apply_sbox, c

    def compute_output(self, state_curr: int, s0: int, s1: int, s2: int) -> int:
        elem = pow5(state_curr) if self.apply_sbox else state_curr
        return (self.q_c + self.coeff * elem + pow5(s0) + s1 + s2) % R


# ---------------------------------------------------------------------------------------------
# The constraint system
# ---------------------------------------------------------------------------------------------
@dataclass
class _Row:
    wires: List[Variable]
    gate: Gate


@dataclass
class GroupLayout:
    """mpc-relation `GroupLayout` (what `get_circuit_layout`, traits.rs:914-946, reports per link group): element i of
    the group sits on wire 0 of the row whose domain point is the (offset + i)-th 2^alignment-th root of unity."""
    alignment: int
    offset: int
    size: int = 0


class PlonkCircuit:
    """mpc-relation `PlonkCircuit<ScalarField>`: variable 0 is the constant zero, variable 1 the constant one
    (each pinned by a constant gate, as upstream's `new()` does)."""

    def __init__(self):
        self.witness_values: List[int] = []
        self.rows: List[_Row] = []
        self.pub_input_vars: List[Variable] = []
        self.link_groups = {}      # id -> (GroupLayout, [variables])
        self._finalized = False
        self._zero = self.create_variable(0)
        self._one = self.create_variable(1)
        self.enforce_constant(self._zero, 0)
        self.enforce_constant(self._one, 1)

    # ---- variables -----------------------------------------------------------------------
    def zero(self) -> Variable:
        return self._zero

    def one(self) -> Variable:
        return self._one

    def create_variable(self, val: int) -> Variable:
        self._check_open()
        self.witness_values.append(val % R)
        return len(self.witness_values) - 1

    def create_public_variable(self, val: int) -> Variable:
        var = self.create_variable(val)
        self.pub_input_vars.append(var)
        self.rows.append(_Row([self._zero] * GATE_WIDTH + [var], IoGate()))
        return var

    def create_link_group(self, group_id: str, layout: GroupLayout) -> str:
        """mpc-relation `create_link_group(id, Some(layout))`: variables added to the group occupy wire 0 of the rows
        the layout names, so that two circuits placing the same values there can be proof-linked
        (`PlonkKzgSnark::link_proofs`, proof_linking/intent_only.rs:42-47)."""
        self._check_open()
        if group_id in self.link_groups:
            raise CircuitError(f"link group {group_id} already exists")
        self.link_groups[group_id] = (GroupLayout(layout.alignment, layout.offset, 0), [])
        return group_id

    def create_variable_with_link_groups(self, val: int, groups: Sequence[str]) -> Variable:
        var = self.create_variable(val)
        for g in groups:
            if g not in self.link_groups:
                raise CircuitError(f"unknown link group {g}")
            layout, members = self.link_groups[g]
            members.append(var)
            layout.size = len(members)
        return var

    def get_circuit_layout(self) -> dict:
        """`get_circuit_layout` (traits.rs:914-946): the placement of every link group."""
        return {g: GroupLayout(l.alignment, l.offset, l.size) for g, (l, _) in self.link_groups.items()}

    def create_constant_variable(self, val: int) -> Variable:
        var = self.create_variable(val)
        self.enforce_constant(var, val)
        return var

    def create_boolean_variable(self, val: bool) -> Variable:
        var = self.create_variable(int(bool(val)))
        self.enforce_bool(var)
        return var

    def witness(self, var: Variable) -> int:
        if not 0 <= var < len(self.witness_values):
            raise CircuitError(f"variable {var} out of bound")
        return self.witness_values[var]

    @property
    def num_vars(self) -> int:
        return len(self.witness_values)

    @property
    def num_gates(self) -> int:
        return len(self.rows)

    @property
    def num_inputs(self) -> int:
        return len(self.pub_input_vars)

    # ---- gates ---------------------------------------------------------------------------
    def insert_gate(self, wire_vars: Sequence[Variable], gate: Gate) -> None:
        self._check_open()
        if len(wire_vars) != GATE_WIDTH + 1:
            raise CircuitError("a gate takes GATE_WIDTH + 1 wires")
        for v in wire_vars:
            self.witness(v)
        self.rows.append(_Row(list(wire_vars), gate))

    def _out(self, wires4: Sequence[Variable], gate: Gate, value: int) -> Variable:
        out = self.create_variable(value)
        self.insert_gate(list(wires4) + [out], gate)
        return out

    def add(self, a: Variable, b: Variable) -> Variable:
        return self._out([a, b, self._zero, self._zero], AdditionGate(), self.witness(a) + self.witness(b))

    def sub(self, a: Variable, b: Variable) -> Variable:
        return self._out([a, b, self._zero, self._zero], SubtractionGate(), self.witness(a) - self.witness(b))

    def mul(self, a: Variable, b: Variable) -> Variable:
        return self._out([a, b, self._zero, self._zero], MultiplicationGate(), self.witness(a) * self.witness(b))

    def lc(self, wires: Sequence[Variable], coeffs: Sequence[int]) -> Variable:
        if len(wires) != GATE_WIDTH or len(coeffs) != GATE_WIDTH:
            raise CircuitError("lc takes GATE_WIDTH wires and coefficients")
        return self._out(wires, LinCombGate(coeffs), sum(c * self.witness(w) for c, w in zip(coeffs, wires)))

    def mux(self, sel: Variable, a: Variable, b: Variable) -> Variable:
        """if sel { a } else { b } (sel must be boolean-constrained by the caller, as `BoolVar` guarantees upstream)."""
        s, va, vb = self.witness(sel), self.witness(a), self.witness(b)
        return self._out([sel, a, sel, b], MuxGate(), s * va + (1 - s) * vb)

    def add_constant(self, a: Variable, c: int) -> Variable:
        return self._out([a, self._zero, self._zero, self._zero], ConstantAdditionGate(c), self.witness(a) + c)

    def lc_sum(self, vars_: Sequence[Variable], coeffs: Sequence[int]) -> Variable:
        """sum_i coeffs[i] * vars[i] with GATE_WIDTH-input linear-combination gates: the first gate takes four terms,
        every further gate the running sum and three more (upstream `lc_sum`)."""
        if len(vars_) != len(coeffs):
            raise CircuitError("lc_sum takes as many coefficients as variables")
        if not vars_:
            return self._zero
        pad = lambda v, c: (list(v) + [self._zero] * (GATE_WIDTH - len(v)), list(c) + [0] * (GATE_WIDTH - len(c)))
        w, c = pad(vars_[:GATE_WIDTH], coeffs[:GATE_WIDTH])
        acc = self.lc(w, c)
        i = GATE_WIDTH
        while i < len(vars_):
            w, c = pad([acc] + list(vars_[i:i + GATE_WIDTH - 1]), [1] + list(coeffs[i:i + GATE_WIDTH - 1]))
            acc = self.lc(w, c)
            i += GATE_WIDTH - 1
        return acc

    def sum(self, vars_: Sequence[Variable]) -> Variable:
        return self.lc_sum(vars_, [1] * len(vars_))

    def mul_gate(self, a: Variable, b: Variable, c: Variable) -> None:
        """enforce a * b = c."""
        self.insert_gate([a, b, self._zero, self._zero, c], MultiplicationGate())

    def mul_add_gate(self, wires: Sequence[Variable], q_mul: Sequence[int]) -> None:
        """enforce q0 * w0 * w1 + q1 * w2 * w3 = w4."""
        self.insert_gate(wires, MulAddGate(q_mul))

    def enforce_true(self, b: Variable) -> None:
        self.enforce_constant(b, 1)

    def enforce_equal(self, a: Variable, b: Variable) -> None:
        self.insert_gate([a, b, self._zero, self._zero, self._zero], EqualityGate())

    def enforce_constant(self, var: Variable, c: int) -> None:
        self.insert_gate([self._zero] * GATE_WIDTH + [var], ConstantGate(c))

    def enforce_bool(self, a: Variable) -> None:
        self.insert_gate([a, a, self._zero, self._zero, a], BoolGate())

    # ---- checks and arithmetization ----------------------------------------------------------
    def _check_open(self) -> None:
        if getattr(self, "_finalized", False):
            raise CircuitError("circuit already finalized for arithmetization")

    def check_circuit_satisfiability(self, pub_inputs: Sequence[int]) -> None:
        """mpc-relation `check_circuit_satisfiability`: every gate equation holds for the current witness, with
        the given public inputs (in `create_public_variable` order) feeding the IO gates."""
        if len(pub_inputs) != self.num_inputs:
            raise CircuitError("wrong number of public inputs")
        pi_of = {id(row): v % R for row, v in zip([r for r in self.rows if r.gate.name == "IoGate"], pub_inputs)}
        for i, row in enumerate(self.rows):
            w = [self.witness_values[v] for v in row.wires]
            if gate_value(row.gate.selectors(), w, pi_of.get(id(row), 0)) != 0:
                raise CircuitError(f"gate {i} ({row.gate.name}) is not satisfied")

    def public_input(self) -> List[int]:
        return [self.witness_values[v] for v in self.pub_input_vars]

    def finalize_for_arithmetization(self, min_log_n: int = 2, wires_only: bool = False,
                                     witness_only: bool = False) -> SynthCircuit:
        """Public-input gates first, zero padding to the next power of two, one copy-constraint cycle per variable
        (upstream: `finalize_for_arithmetization`, traits.rs:847,991).  Returns the flat tables the C ABI takes.

        Layout / verifying-key parity with the Rust reference is NOT claimed: this places the public-input gates by a
        stable partition (io + rest) and uses coset representatives k_i = 5^i, while the un-vendored jellyfish fork may
        swap gate i with IO gate i and derives k from its own generator.  Proofs made here are self-consistent and
        verify under the key preprocessed from the same tables; a production host passes the Rust-built selector /
        permutation tables and `vk.k` through the ABI (INTEGRATION.md section 2), so the layout is the reference's."""
        self._check_open()
        io = [r for r in self.rows if r.gate.name == "IoGate"]
        rest = [r for r in self.rows if r.gate.name != "IoGate"]
        n_link = sum(len(m) for _, m in self.link_groups.values())
        n_gates = len(io) + len(rest) + n_link
        log_n = max([min_log_n, (n_gates - 1).bit_length()] + [l.alignment for l, _ in self.link_groups.values()])
        while True:  # link rows are pinned to domain positions; everything else flows around them
            n = 1 << log_n
            pinned = {}
            for gid, (l, members) in self.link_groups.items():
                for i, var in enumerate(members):
                    row = (l.offset + i) << (log_n - l.alignment)
                    if row >= n or row < len(io) or row in pinned:
                        raise CircuitError(f"link group {gid}: row {row} is outside the domain or already taken")
                    pinned[row] = var
            if n - len(pinned) >= len(io) + len(rest):
                break
            log_n += 1
        rows: List[_Row] = []
        pending = iter(io + rest)
        for r in range(n):
            if r in pinned:  # link gate: the value on wire 0, no constraint of its own
                rows.append(_Row([pinned[r]] + [self._zero] * GATE_WIDTH, Gate("LinkGate")))
            else:
                rows.append(next(pending, None) or _Row([self._zero] * (GATE_WIDTH + 1), PaddingGate()))
        # `wires_only` (f4 of SURVEY 8(f): the structure is witness-independent and lives in the preprocessed key; per proof
        # only the 5 x n value table changes): skip the selector columns and the copy permutation, keep their fingerprint
        gate_sels = [tuple(row.gate.selectors()) for row in rows]
        digest = hash((n, tuple(tuple(row.wires) for row in rows), tuple(gate_sels))) or 1
        # `witness_only` (a key made by `preprocess_wiring` holds the wiring too): per proof only the witness vector goes
        # to the device, and the 5 x n value table is never built on the host
        if witness_only:
            pub = self.public_input()
            self._finalized = True
            return SynthCircuit(log_n=log_n, num_inputs=len(pub), k=to_mont_array([pow(5, i, R) for i in range(N_WIRES)]),
                                selectors=None, perm=None, wires=None, pub_inputs=to_mont_array(pub), n_gates=n_gates,
                                selectors_int=None, wires_int=None, pub_inputs_int=pub, structure_digest=digest,
                                witness=to_mont_array(self.witness_values))
        wires_int = [[self.witness_values[row.wires[w]] for row in rows] for w in range(N_WIRES)]
        pub = self.public_input()
        k_int = [pow(5, i, R) for i in range(N_WIRES)]
        wires = np.stack([to_mont_array(col) for col in wires_int])
        pub_arr = to_mont_array(pub) if pub else np.zeros((0, 4), dtype=np.uint64)
        self._finalized = True
        if wires_only:
            return SynthCircuit(log_n=log_n, num_inputs=len(pub), k=to_mont_array(k_int), selectors=None, perm=None,
                                wires=wires, pub_inputs=pub_arr, n_gates=n_gates, selectors_int=None, wires_int=wires_int,
                                pub_inputs_int=pub, structure_digest=digest)
        sel = [[q[s] for q in gate_sels] for s in range(N_SELECTORS)]
        positions: List[List] = [[] for _ in self.witness_values]
        for r, row in enumerate(rows):
            for wcol, var in enumerate(row.wires):
                positions[var].append((wcol, r))
        perm = np.empty(N_WIRES * n, dtype=np.uint64)
        for occ in positions:
            for a, b in zip(occ, occ[1:] + occ[:1]):
                perm[a[0] * n + a[1]] = b[0] * n + b[1]
        return SynthCircuit(log_n=log_n, num_inputs=len(pub), k=to_mont_array(k_int),
                            selectors=np.stack([to_mont_array(col) for col in sel]), perm=perm, wires=wires,
                            pub_inputs=pub_arr, n_gates=n_gates, selectors_int=sel, wires_int=wires_int, pub_inputs_int=pub,
                            structure_digest=digest,
                            wire_vars=np.array([row.wires for row in rows], dtype=np.uint32).T.copy(),
                            witness=to_mont_array(self.witness_values))


# ---------------------------------------------------------------------------------------------
# Native Poseidon2 (witness side)
# ---------------------------------------------------------------------------------------------
def _external_mds(s: List[int]) -> List[int]:
    t = sum(s) % R
    return [(x + t) % R for x in s]


def _internal_mds(s: List[int]) -> List[int]:
    t = sum(s) % R
    return [(s[0] + t) % R, (s[1] + t) % R, (2 * s[2] + t) % R]


class Poseidon2Sponge:
    """crates/crypto/src/hash/poseidon2.rs:25-209: width 3, rate 2, capacity 1, R_F = 8, R_P = 56, alpha = 5."""

    def __init__(self):
        self.state = [0] * (CAPACITY + RATE)
        self.next_index = 0
        self.squeezing = False

    def permute(self) -> None:
        st = _external_mds(self.state)
        half = R_F // 2
        for r in range(half):
            st = _external_mds([pow5((x + FULL_ROUND_CONSTANTS[r][i]) % R) for i, x in enumerate(st)])
        for r in range(R_P):
            st = _internal_mds([pow5((st[0] + PARTIAL_ROUND_CONSTANTS[r]) % R), st[1], st[2]])
        for r in range(half, R_F):
            st = _external_mds([pow5((x + FULL_ROUND_CONSTANTS[r][i]) % R) for i, x in enumerate(st)])
        self.state = st

    def absorb(self, x: int) -> None:
        if self.squeezing:
            raise ValueError("cannot absorb while squeezing")
        if self.next_index == RATE:
            self.permute()
            self.next_index = 0
        self.state[self.next_index + CAPACITY] = (self.state[self.next_index + CAPACITY] + x) % R
        self.next_index += 1

    def absorb_batch(self, xs: Sequence[int]) -> None:
        for x in xs:
            self.absorb(x)

    def squeeze(self) -> int:
        if not self.squeezing or self.next_index == RATE:
            self.permute()
            self.next_index = 0
            self.squeezing = True
        out = self.state[self.next_index + CAPACITY]
        self.next_index += 1
        return out

    def hash(self, xs: Sequence[int]) -> int:
        self.absorb_batch(xs)
        return self.squeeze()


def compute_poseidon_hash(values: Sequence[int]) -> int:
    """crates/crypto/src/hash/mod.rs:12-18."""
    return Poseidon2Sponge().hash(values)


# ---------------------------------------------------------------------------------------------
# Gadgets
# ---------------------------------------------------------------------------------------------
class PoseidonHashGadget:
    """poseidon/hash.rs:56-423: the sponge over circuit variables; a permutation is 195 gates (one external MDS,
    8 fused external rounds, 56 fused internal rounds, 3 gates each), every gate carrying the NEXT round's constant."""

    def __init__(self, zero_var: Variable):
        self.state = [zero_var] * (CAPACITY + RATE)
        self.next_index = 0
        self.in_squeeze_state = False

    def clone(self) -> "PoseidonHashGadget":
        other = PoseidonHashGadget(self.state[0])
        other.state, other.next_index, other.in_squeeze_state = list(self.state), self.next_index, self.in_squeeze_state
        return other

    def reset_state(self, cs: PlonkCircuit) -> None:
        self.state = [cs.zero()] * (CAPACITY + RATE)
        self.next_index = 0
        self.in_squeeze_state = False

    def hash(self, hash_input: Sequence[Variable], cs: PlonkCircuit) -> Variable:
        self.batch_absorb(hash_input, cs)
        return self.squeeze(cs)

    def hash_constrained(self, hash_input: Sequence[Variable], expected_output: Variable, cs: PlonkCircuit) -> None:
        self.batch_absorb(hash_input, cs)
        self.constrained_squeeze(expected_output, cs)

    def absorb(self, a: Variable, cs: PlonkCircuit) -> None:
        if self.in_squeeze_state:
            raise CircuitError("Cannot absorb from a sponge that has already been squeezed")
        if self.next_index == RATE:
            self.permute(cs)
            self.next_index = 0
        idx = self.next_index + CAPACITY
        self.state[idx] = cs.add(a, self.state[idx])
        self.next_index += 1

    def batch_absorb(self, xs: Sequence[Variable], cs: PlonkCircuit) -> None:
        for x in xs:
            self.absorb(x, cs)

    def squeeze(self, cs: PlonkCircuit) -> Variable:
        if not self.in_squeeze_state or self.next_index == RATE:
            self.permute(cs)
            self.next_index = 0
            self.in_squeeze_state = True
        res = self.state[CAPACITY + self.next_index]
        self.next_index += 1
        return res

    def batch_squeeze(self, num_elements: int, cs: PlonkCircuit) -> List[Variable]:
        return [self.squeeze(cs) for _ in range(num_elements)]

    def constrained_squeeze(self, expected: Variable, cs: PlonkCircuit) -> None:
        cs.enforce_equal(expected, self.squeeze(cs))

    # ---- permutation (hash.rs:205-262) ------------------------------------------------------
    def permute(self, cs: PlonkCircuit) -> None:
        half = R_F // 2
        self._fused_external(False, FULL_ROUND_CONSTANTS[0], cs)
        for rnd in range(half - 1):
            self._fused_external(True, FULL_ROUND_CONSTANTS[rnd + 1], cs)
        rc = [PARTIAL_ROUND_CONSTANTS[0], 0, 0]
        self._fused_external(True, rc, cs)
        for rnd in range(R_P - 1):
            rc[0] = PARTIAL_ROUND_CONSTANTS[rnd + 1]
            self._fused_internal(rc, cs)
        self._fused_internal(FULL_ROUND_CONSTANTS[half], cs)
        for rnd in range(half, R_F - 1):
            self._fused_external(True, FULL_ROUND_CONSTANTS[rnd + 1], cs)
        self._fused_external(True, [0, 0, 0], cs)

    def _fused_external(self, apply_sbox: bool, next_round_const: Sequence[int], cs: PlonkCircuit) -> None:
        in_wires = list(self.state)
        vals = [cs.witness(v) for v in in_wires]
        for i in range(3):
            gate = FusedExternalSboxMDSGate(apply_sbox, next_round_const[i])
            out = cs.create_variable(gate.compute_output(vals[i], *vals))
            cs.insert_gate([in_wires[i]] + in_wires + [out], gate)
            self.state[i] = out

    def _fused_internal(self, next_round_constants: Sequence[int], cs: PlonkCircuit) -> None:
        in_wires = list(self.state)
        vals = [cs.witness(v) for v in in_wires]
        for i, (sbox, coeff) in enumerate(((True, 1), (False, 1), (False, 2))):
            gate = FusedInternalSboxMDSGate(sbox, next_round_constants[i], coeff)
            out = cs.create_variable(gate.compute_output(vals[i], *vals))
            cs.insert_gate([in_wires[i]] + in_wires + [out], gate)
            self.state[i] = out


def scalar_to_bits_le(a: int, n: int) -> List[int]:
    """bits.rs:12-21: the low n bits, little-endian (zero-extended)."""
    return [(a >> i) & 1 for i in range(n)]


class ToBitsGadget:
    """bits.rs:22-78."""

    @staticmethod
    def to_bits(a: Variable, num_bits: int, cs: PlonkCircuit) -> List[Variable]:
        bits = [cs.create_boolean_variable(b) for b in scalar_to_bits_le(cs.witness(a), num_bits)]
        cs.enforce_equal(ToBitsGadget.bit_reconstruct(bits, cs), a)
        return bits

    @staticmethod
    def bit_reconstruct(bits: Sequence[Variable], cs: PlonkCircuit) -> Variable:
        return cs.lc_sum(bits, [1 << i for i in range(len(bits))])


class BitRangeGadget:
    """bits.rs:80-95: a in [0, 2^num_bits)."""

    @staticmethod
    def constrain_bit_range(a: Variable, num_bits: int, cs: PlonkCircuit) -> None:
        ToBitsGadget.to_bits(a, num_bits, cs)


class EqZeroGadget:
    """comparators.rs:17-60: is_zero = 1 - val * inv and is_zero * val = 0."""

    @staticmethod
    def eq_zero_var(val: Variable, cs: PlonkCircuit) -> Variable:
        v = cs.witness(val)
        is_zero = cs.create_variable(1 if v == 0 else 0)
        inv = cs.create_variable(0 if v == 0 else pow(v, -1, R))
        cs.mul_add_gate([val, inv, cs.one(), cs.one(), is_zero], [-1, 1])
        cs.mul_gate(is_zero, val, cs.zero())
        return is_zero


class GreaterThanEqZeroGadget:
    """comparators.rs:183-234: for x in [-2^D, 2^D), x >= 0 iff bit D of x + 2^D is set."""

    @staticmethod
    def greater_than_eq_zero(x: Variable, num_bits: int, cs: PlonkCircuit) -> Variable:
        shifted = cs.add_constant(x, 1 << num_bits)
        return ToBitsGadget.to_bits(shifted, num_bits + 1, cs)[num_bits]

    @staticmethod
    def constrain_greater_than_eq_zero(x: Variable, num_bits: int, cs: PlonkCircuit) -> None:
        ToBitsGadget.to_bits(x, num_bits, cs)


class GreaterThanEqGadget:
    """comparators.rs:236-262: a >= b for values of at most num_bits bits."""

    @staticmethod
    def greater_than_eq(a: Variable, b: Variable, num_bits: int, cs: PlonkCircuit) -> Variable:
        return GreaterThanEqZeroGadget.greater_than_eq_zero(cs.sub(a, b), num_bits, cs)

    @staticmethod
    def constrain_greater_than_eq(a: Variable, b: Variable, num_bits: int, cs: PlonkCircuit) -> None:
        GreaterThanEqZeroGadget.constrain_greater_than_eq_zero(cs.sub(a, b), num_bits, cs)


# ---- state primitives: CSPRNG streams, stream cipher, recovery ids, commitments ---------------------------
AMOUNT_BITS = 100  # circuit-types/src/lib.rs:59


@dataclass
class PoseidonCSPRNG:
    """darkpool-types/src/csprng.rs:30-75: value i of the stream is H(seed, i)."""
    seed: int
    index: int = 0

    def next(self) -> int:
        out = compute_poseidon_hash([self.seed, self.index])
        self.index += 1
        return out

    def get_ith(self, i: int) -> int:
        return compute_poseidon_hash([self.seed, i])

    def to_scalars(self) -> List[int]:
        return [self.seed, self.index]

    def stream_cipher_encrypt(self, values: Sequence[int]) -> List[int]:
        """csprng.rs:62-74: ciphertext = value - pad, one fresh pad per value."""
        return [(v - self.next()) % R for v in values]


@dataclass
class StateWrapper:
    """darkpool-types/src/state_wrapper.rs:60-190 for an element given as its scalar serialisation."""
    recovery_stream: PoseidonCSPRNG
    share_stream: PoseidonCSPRNG
    inner: List[int]
    public_share: List[int]

    @staticmethod
    def new(inner: Sequence[int], share_stream_seed: int, recovery_stream_seed: int) -> "StateWrapper":
        share = PoseidonCSPRNG(share_stream_seed)
        public = share.stream_cipher_encrypt(inner)
        return StateWrapper(PoseidonCSPRNG(recovery_stream_seed), share, list(inner), public)

    def private_shares(self) -> List[int]:
        return [(v - p) % R for v, p in zip(self.inner, self.public_share)]

    def compute_recovery_id(self) -> int:
        return self.recovery_stream.next()

    def compute_private_commitment(self) -> int:
        return compute_poseidon_hash(self.private_shares() + self.recovery_stream.to_scalars() + self.share_stream.to_scalars())

    def compute_commitment(self) -> int:
        return compute_poseidon_hash([self.compute_private_commitment(), self.compute_partial_public_commitment(len(self.public_share))])

    def compute_partial_public_commitment(self, num_shares: int) -> int:
        """state_wrapper.rs:133-142: the resumable chain over the first `num_shares` public shares."""
        comm = self.public_share[0]
        for share in self.public_share[1:num_shares]:
            comm = compute_poseidon_hash([comm, share])
        return comm

    def compute_partial_commitment(self, num_shares: int):
        """state_wrapper.rs:104-108: (private commitment, partial public commitment)."""
        return self.compute_private_commitment(), self.compute_partial_public_commitment(num_shares)

    def compute_nullifier(self) -> int:
        """state_wrapper.rs:146-154: H(last recovery id, recovery stream seed)."""
        return compute_poseidon_hash([self.recovery_stream.get_ith(self.recovery_stream.index - 1), self.recovery_stream.seed])

    def clone(self) -> "StateWrapper":
        return StateWrapper(PoseidonCSPRNG(self.recovery_stream.seed, self.recovery_stream.index),
                            PoseidonCSPRNG(self.share_stream.seed, self.share_stream.index), list(self.inner), list(self.public_share))


@dataclass
class PoseidonCSPRNGVar:
    seed: Variable
    index: Variable

    def to_vars(self) -> List[Variable]:
        return [self.seed, self.index]

    def clone(self) -> "PoseidonCSPRNGVar":
        return PoseidonCSPRNGVar(self.seed, self.index)


@dataclass
class StateWrapperVar:
    """darkpool-types `StateWrapperVar<T>`: the element's variables with its two stream states and public shares."""
    recovery_stream: PoseidonCSPRNGVar
    share_stream: PoseidonCSPRNGVar
    inner: List[Variable]
    public_share: List[Variable]

    def clone(self) -> "StateWrapperVar":
        return StateWrapperVar(self.recovery_stream.clone(), self.share_stream.clone(), list(self.inner), list(self.public_share))

    @staticmethod
    def create_witness(w: "StateWrapper", cs: PlonkCircuit) -> "StateWrapperVar":
        mk = lambda st: PoseidonCSPRNGVar(cs.create_variable(st.seed), cs.create_variable(st.index))
        return StateWrapperVar(mk(w.recovery_stream), mk(w.share_stream), [cs.create_variable(v) for v in w.inner],
                               [cs.create_variable(v) for v in w.public_share])


class CSPRNGGadget:
    """state_primitives/csprng.rs:9-47."""

    @staticmethod
    def get_ith(state: PoseidonCSPRNGVar, i: Variable, cs: PlonkCircuit) -> Variable:
        return PoseidonHashGadget(cs.zero()).hash([state.seed, i], cs)

    @staticmethod
    def next(state: PoseidonCSPRNGVar, cs: PlonkCircuit) -> Variable:
        value = PoseidonHashGadget(cs.zero()).hash([state.seed, state.index], cs)
        state.index = cs.add(state.index, cs.one())
        return value

    @staticmethod
    def next_k(state: PoseidonCSPRNGVar, k: int, cs: PlonkCircuit) -> List[Variable]:
        return [CSPRNGGadget.next(state, cs) for _ in range(k)]


class StreamCipherGadget:
    """state_primitives/stream_cipher.rs:13-33: returns (private share = the pads, public share = value - pad)."""

    @staticmethod
    def encrypt(value_vars: Sequence[Variable], state: PoseidonCSPRNGVar, cs: PlonkCircuit):
        pads = CSPRNGGadget.next_k(state, len(value_vars), cs)
        return pads, [cs.sub(v, p) for v, p in zip(value_vars, pads)]


class RecoveryIdGadget:
    """state_primitives/recovery_id.rs:9-20."""

    @staticmethod
    def compute_recovery_id(recovery_stream: PoseidonCSPRNGVar, cs: PlonkCircuit) -> Variable:
        return CSPRNGGadget.next(recovery_stream, cs)


class CommitmentGadget:
    """state_primitives/commitment.rs:33-95, 433-446."""

    @staticmethod
    def compute_commitment(private_share: Sequence[Variable], recovery_stream: PoseidonCSPRNGVar,
                           share_stream: PoseidonCSPRNGVar, public_share: Sequence[Variable], cs: PlonkCircuit) -> Variable:
        hasher = PoseidonHashGadget(cs.zero())
        hasher.batch_absorb(list(private_share) + recovery_stream.to_vars() + share_stream.to_vars(), cs)
        private_commitment = hasher.squeeze(cs)
        public_commitment = CommitmentGadget.compute_resumable_commitment(public_share, cs)
        return PoseidonHashGadget(cs.zero()).hash([private_commitment, public_commitment], cs)

    @staticmethod
    def compute_resumable_commitment(values: Sequence[Variable], cs: PlonkCircuit) -> Variable:
        if not values:
            raise CircuitError("Cannot compute a resumable commitment with no values")
        comm = values[0]
        for value in values[1:]:
            comm = PoseidonHashGadget(cs.zero()).hash([comm, value], cs)
        return comm


def _shared_prefix_length(a: Sequence[Variable], b: Sequence[Variable]) -> int:
    """commitment.rs:14-29: how many leading VARIABLES two share vectors have in common."""
    n = 0
    while n < len(a) and a[n] == b[n]:
        n += 1
    return n


class SharedPrefixCommitmentGadget:
    """commitment.rs:128-330: commitments to two versions of an element that share a prefix of their shares hash that
    prefix once (the new version of a rotated element differs from the old one in a few trailing fields only)."""

    @staticmethod
    def compute_private_commitments(priv1, priv2, elt1: "StateWrapperVar", elt2: "StateWrapperVar", cs: PlonkCircuit):
        k = _shared_prefix_length(priv1, priv2)
        hasher = PoseidonHashGadget(cs.zero())
        hasher.batch_absorb(list(priv1[:k]), cs)
        out = []
        for priv, elt in ((priv1, elt1), (priv2, elt2)):
            h = hasher.clone()
            h.batch_absorb(list(priv[k:]) + elt.recovery_stream.to_vars() + elt.share_stream.to_vars(), cs)
            out.append(h.squeeze(cs))
        return out[0], out[1]

    @staticmethod
    def compute_public_partial_commitments(num_shares: int, pub1, pub2, cs: PlonkCircuit):
        k = min(_shared_prefix_length(pub1, pub2), num_shares)
        v1, v2 = [], []
        if k > 0:
            partial = CommitmentGadget.compute_resumable_commitment(list(pub1[:k]), cs)
            v1, v2 = [partial], [partial]
        v1 += list(pub1[k:])
        v2 += list(pub2[k:num_shares])
        return CommitmentGadget.compute_resumable_commitment(v1, cs), CommitmentGadget.compute_resumable_commitment(v2, cs)

    @staticmethod
    def compute_partial_commitments(num_shares: int, priv1, elt1, priv2, elt2, cs: PlonkCircuit):
        """-> (full commitment of element 1, (private commitment, partial public commitment) of element 2)."""
        pc1, pc2 = SharedPrefixCommitmentGadget.compute_private_commitments(priv1, priv2, elt1, elt2, cs)
        pub1, pub2 = SharedPrefixCommitmentGadget.compute_public_partial_commitments(num_shares, elt1.public_share,
                                                                                      elt2.public_share, cs)
        return PoseidonHashGadget(cs.zero()).hash([pc1, pub1], cs), (pc2, pub2)


class NotEqualGadget:
    """comparators.rs:143-170: a != b as 1 - (a - b == 0), constrained true."""

    @staticmethod
    def constrain_not_equal(a: Variable, b: Variable, cs: PlonkCircuit) -> None:
        eq = EqZeroGadget.eq_zero_var(cs.sub(a, b), cs)
        neq = cs.lc([cs.one(), eq, cs.zero(), cs.zero()], [1, -1, 0, 0])
        cs.enforce_true(neq)


class NullifierGadget:
    """state_primitives/nullifier.rs:10-33: H(recovery id of the last update, recovery stream seed)."""

    @staticmethod
    def compute_nullifier(element: "StateWrapperVar", cs: PlonkCircuit) -> Variable:
        NotEqualGadget.constrain_not_equal(element.recovery_stream.index, cs.zero(), cs)
        last_idx = cs.sub(element.recovery_stream.index, cs.one())
        recovery_id = CSPRNGGadget.get_ith(element.recovery_stream, last_idx, cs)
        return PoseidonHashGadget(cs.zero()).hash([recovery_id, element.recovery_stream.seed], cs)


class ShareGadget:
    """state_primitives/shares.rs:17-60."""

    @staticmethod
    def compute_complementary_shares(shares: Sequence[Variable], base: Sequence[Variable], cs: PlonkCircuit) -> List[Variable]:
        return [cs.sub(b, s) for b, s in zip(base, shares)]


class StateElementRotationGadget:
    """state_primitives/state_rotation.rs:97-140 (`rotate_version_with_partial_commitment`): the new version's
    recovery id, the old version's full and the new version's partial commitment (shared prefix), the Merkle opening
    of the old commitment, the old version's nullifier."""

    @staticmethod
    def rotate_version_with_partial_commitment(num_shares: int, old_version: "StateWrapperVar", old_private_share,
                                               old_opening: "MerkleOpeningVar", merkle_root: Variable, nullifier: Variable,
                                               new_version: "StateWrapperVar", new_private_share,
                                               new_partial_commitment, recovery_id: Variable, cs: PlonkCircuit) -> None:
        cs.enforce_equal(RecoveryIdGadget.compute_recovery_id(new_version.recovery_stream, cs), recovery_id)
        old_commitment, (priv_c, pub_c) = SharedPrefixCommitmentGadget.compute_partial_commitments(
            num_shares, old_private_share, old_version, new_private_share, new_version, cs)
        cs.enforce_equal(priv_c, new_partial_commitment[0])
        cs.enforce_equal(pub_c, new_partial_commitment[1])
        root = PoseidonMerkleHashGadget.compute_root_prehashed(old_commitment, old_opening, cs)
        cs.enforce_equal(merkle_root, root)
        cs.enforce_equal(NullifierGadget.compute_nullifier(old_version, cs), nullifier)


    @staticmethod
    def rotate_version(old_version: "StateWrapperVar", old_private_share, old_opening: "MerkleOpeningVar",
                       merkle_root: Variable, nullifier: Variable, new_version: "StateWrapperVar", new_private_share,
                       new_commitment: Variable, recovery_id: Variable, cs: PlonkCircuit) -> None:
        """state_rotation.rs:81-121 (`rotate_version`): as above with the FULL commitment of the new version
        (commitment.rs:193-224, `compute_commitments_with_shared_prefix`: both public chains run to the end)."""
        cs.enforce_equal(RecoveryIdGadget.compute_recovery_id(new_version.recovery_stream, cs), recovery_id)
        pc_old, pc_new = SharedPrefixCommitmentGadget.compute_private_commitments(old_private_share, new_private_share,
                                                                                  old_version, new_version, cs)
        pub_old, pub_new = SharedPrefixCommitmentGadget.compute_public_partial_commitments(
            len(new_version.public_share), old_version.public_share, new_version.public_share, cs)
        old_commitment = PoseidonHashGadget(cs.zero()).hash([pc_old, pub_old], cs)
        cs.enforce_equal(PoseidonHashGadget(cs.zero()).hash([pc_new, pub_new], cs), new_commitment)
        root = PoseidonMerkleHashGadget.compute_root_prehashed(old_commitment, old_opening, cs)
        cs.enforce_equal(merkle_root, root)
        cs.enforce_equal(NullifierGadget.compute_nullifier(old_version, cs), nullifier)


class AmountGadget:
    """primitives/bitlength.rs:9-17."""

    @staticmethod
    def constrain_valid_amount(amount: Variable, cs: PlonkCircuit) -> None:
        BitRangeGadget.constrain_bit_range(amount, AMOUNT_BITS, cs)


@dataclass
class MerkleOpening:
    """circuit-types `MerkleOpening<HEIGHT>`: sister nodes bottom-up and, per level, whether the running hash is the
    RIGHT child of its parent."""
    elems: List[int]
    indices: List[bool]


@dataclass
class MerkleOpeningVar:
    elems: List[Variable] = field(default_factory=list)
    indices: List[Variable] = field(default_factory=list)


class PoseidonMerkleHashGadget:
    """primitives/merkle.rs:13-126."""

    @staticmethod
    def compute_root(leaf_node: Sequence[Variable], opening: MerkleOpeningVar, cs: PlonkCircuit) -> Variable:
        leaf_hash = PoseidonHashGadget(cs.zero()).hash(leaf_node, cs)
        return PoseidonMerkleHashGadget.compute_root_prehashed(leaf_hash, opening, cs)

    @staticmethod
    def compute_root_prehashed(leaf_node: Variable, opening: MerkleOpeningVar, cs: PlonkCircuit) -> Variable:
        current = leaf_node
        for path_elem, lr_select in zip(opening.elems, opening.indices):
            # lr_select is true when the running hash is the right child (merkle.rs:80-91)
            left = cs.mux(lr_select, path_elem, current)
            right = cs.lc([current, path_elem, left, cs.zero()], [1, 1, -1, 1])
            current = PoseidonHashGadget(cs.zero()).hash([left, right], cs)
        return current

    @staticmethod
    def compute_and_constrain_root(leaf_node: Sequence[Variable], opening: MerkleOpeningVar, expected_root: Variable,
                                   cs: PlonkCircuit) -> None:
        cs.enforce_equal(expected_root, PoseidonMerkleHashGadget.compute_root(leaf_node, opening, cs))


def native_merkle_root_prehashed(leaf_hash: int, opening: MerkleOpening) -> int:
    cur = leaf_hash
    for sister, is_right in zip(opening.elems, opening.indices):
        cur = compute_poseidon_hash([sister, cur] if is_right else [cur, sister])
    return cur


def native_merkle_root(leaf: Sequence[int], opening: MerkleOpening) -> int:
    """The root `PoseidonMerkleHashGadget::compute_root` constrains, computed natively (merkle.rs tests: leaf hash =
    sponge over the leaf buffer, internal nodes = two-to-one sponge hashes)."""
    cur = compute_poseidon_hash(leaf)
    for sister, is_right in zip(opening.elems, opening.indices):
        cur = compute_poseidon_hash([sister, cur] if is_right else [cur, sister])
    return cur


def merkle_membership_circuit(leaf: Sequence[int], opening: MerkleOpening):
    """A statement of the reference's shape in miniature: the Merkle root is public (like `merkle_root` in the
    VALID-* statements), the leaf buffer and its opening are the witness.  Returns (PlonkCircuit, root)."""
    cs = PlonkCircuit()
    root_val = native_merkle_root(leaf, opening)
    root = cs.create_public_variable(root_val)
    leaf_vars = [cs.create_variable(v) for v in leaf]
    op = MerkleOpeningVar([cs.create_variable(v) for v in opening.elems],
                          [cs.create_boolean_variable(b) for b in opening.indices])
    PoseidonMerkleHashGadget.compute_and_constrain_root(leaf_vars, op, root, cs)
    return cs, root_val
