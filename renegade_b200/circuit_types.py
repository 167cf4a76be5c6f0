"""`SingleProverCircuit` surface over the GPU proving backend — the host-side mirror of
/root/reference/crates/circuits/circuit-types/src/traits.rs:75-92, 817-1020 and
circuits-core/src/lib.rs:112-142, so that callers (and the parity tests) read like the reference's:

    proof          = singleprover_prove(ValidBalanceCreate, witness, statement)
    proof, hint    = singleprover_prove_with_hint(C, witness, statement)
    proofs         = singleprover_prove_batch(C, [(witness, statement), ...])   # one batch call on the device
    verify_singleprover_proof(C, statement, proof)         # raises VerifierError
    singleprover_prove_and_verify(C, witness, statement)

What this module owns (the reference's `circuit-types` side of the boundary):
  * `SYSTEM_SRS` (`set_system_srs`): the G1 powers resident on the device + the two G2 elements of the open key;
  * the proving/verifying key cache keyed by `C.name()` (`setup_preprocessed_keys`, traits.rs:821-855: keys are derived
    once per circuit from a dummy instance of the right topology and shared by every prover thread) and the circuit
    layout cache (traits.rs:914-946);
  * prove = synthesise -> finalize -> draw the 17 blinders from the OS RNG (`thread_rng()`, traits.rs:994) ->
    `PlonkKzgSnark.prove_with_link_hint` (device); verify = statement scalars -> `PlonkKzgSnark.verify` (host pairing);
  * the error split `ProverError::{Circuit, Plonk, Verification}` / `VerifierError::Plonk` (errors.rs:33-58).

What it does NOT own: the constraint system.  mpc-relation's `PlonkCircuit` and the gadgets are upstream / caller code
(Rust in a deployment; the Python restatement under examples/host_circuits for tests and benches).  A circuit class
therefore provides `synthesize(witness, statement, layout)` returning any object with `finalize_for_arithmetization()`
(-> tables in the layout of `renegade_b200.synth.SynthCircuit`) and, for link groups, `get_circuit_layout()`.
"""
from __future__ import annotations

import os
import threading
from dataclasses import dataclass
from typing import Any, Dict, List, Optional, Tuple

import numpy as np

from . import _lib
from .backend import (B200Proof, Bases, Context, GroupLayout, LinkingHint, PlonkKzgSnark, ProvingKey, VerifyingKey, check_srs,
                      parse_ptau_file, read_ptau_g2)
from .fields import SCALAR_FIELD_MODULUS, scalars_to_limbs

PlonkProof = B200Proof                    # circuit-types/src/lib.rs:72-101
ProofLinkingHint = LinkingHint


class ProverError(Exception):
    """circuit-types/src/errors.rs:33-47.  `kind` is one of "Circuit", "Plonk", "Verification", or "Srs" (an SRS that
    failed `SystemSrs.from_ptau`'s check; `detail` is its SrsReport)."""

    def __init__(self, kind: str, detail: Any):
        super().__init__(f"{kind}({detail})")
        self.kind, self.detail = kind, detail


class VerifierError(Exception):
    """circuit-types/src/errors.rs:50-58 (`VerifierError::Plonk`)."""


@dataclass
class SystemSrs:
    """`SYSTEM_SRS` (primitives/srs.rs:30-71): `powers_of_g` on the device, `h` / `beta_h` as 128-byte G2 records."""
    ctx: Context
    powers_of_g: Bases
    g2_h: np.ndarray
    g2_tau_h: np.ndarray
    pool: Any = None   # optional ProverPool: proofs then run `workers` at a time, one request thread per ticket

    @staticmethod
    def from_ptau(ctx: Context, data: bytes, count: Optional[int] = None, check: bool = True, pool=None) -> "SystemSrs":
        """The whole SRS from one ptau file: the G1 powers (`count` of them, default MAX_SRS_DEGREE + 1) loaded on the
        device, h / beta_h from its section 3, and with `check` the powers checked against them on the device
        (`check_srs`, fresh random weights); then installed as SYSTEM_SRS (`set_system_srs`).  An SRS that fails the
        check raises ProverError("Srs", report) and nothing is installed."""
        params = parse_ptau_file(ctx, data, count=count)
        h, beta_h = (params.h, params.beta_h) if params.h is not None else read_ptau_g2(data)
        if check:
            report = check_srs(ctx, params.powers_of_g, h, beta_h)
            if not report.valid:
                params.powers_of_g.free()
                raise ProverError("Srs", report)
        return set_system_srs(ctx, params.powers_of_g, h, beta_h, pool=pool)


_SYSTEM_SRS: Optional[SystemSrs] = None
_KEY_LOCK = threading.RLock()
_CIRCUIT_KEY_CACHE: Dict[str, Tuple[ProvingKey, VerifyingKey]] = {}
_CIRCUIT_LAYOUT_CACHE: Dict[str, Any] = {}
_CIRCUIT_STRUCTURE: Dict[str, int] = {}  # name -> fingerprint of the structure its key was preprocessed from (0: unknown)


def set_system_srs(ctx: Context, powers_of_g: Bases, g2_h: np.ndarray, g2_tau_h: np.ndarray, pool=None) -> SystemSrs:
    """Install the process-wide SRS (the reference parses srs/srs00 once, lazily).  Clears the key cache: keys
    belong to the SRS they were derived from.  `pool` (a `ProverPool` on the same device, whose worker-0 context is
    `ctx`): proofs are queued there — the shape of `NativeProofManager`'s rayon pool — instead of serialising on `ctx`."""
    global _SYSTEM_SRS
    with _KEY_LOCK:
        clear_key_cache()
        _SYSTEM_SRS = SystemSrs(ctx, powers_of_g, np.ascontiguousarray(g2_h, dtype=np.uint64).reshape(16),
                                np.ascontiguousarray(g2_tau_h, dtype=np.uint64).reshape(16), pool)
        return _SYSTEM_SRS


def system_srs() -> SystemSrs:
    if _SYSTEM_SRS is None:
        raise ProverError("Plonk", "SYSTEM_SRS is not set (call set_system_srs)")
    return _SYSTEM_SRS


def clear_key_cache() -> None:
    with _KEY_LOCK:
        for pk, _ in _CIRCUIT_KEY_CACHE.values():
            try:
                pk.free()
            except Exception:
                pass
        _CIRCUIT_KEY_CACHE.clear()
        _CIRCUIT_LAYOUT_CACHE.clear()
        _CIRCUIT_STRUCTURE.clear()


def draw_blinders(rng=None) -> np.ndarray:
    """The 17 field elements the prover draws (2 per wire polynomial, 3 for the permutation product, 4 for the quotient
    split), Montgomery form.  rng = None: the OS generator, as `thread_rng()` at traits.rs:994; a `random.Random` makes
    a proof reproducible (the parity tests do that on both sides)."""
    if rng is None:
        vals = [int.from_bytes(os.urandom(48), "little") % SCALAR_FIELD_MODULUS for _ in range(17)]  # 384 bits: negligible bias
    else:
        vals = [rng.randrange(SCALAR_FIELD_MODULUS) for _ in range(17)]
    return scalars_to_limbs(vals)


def setup_preprocessed_keys(circuit: type) -> Tuple[ProvingKey, VerifyingKey]:
    """traits.rs:821-855: keys from the cache, else derived from a dummy instance of the circuit's topology."""
    name = circuit.name()
    with _KEY_LOCK:
        hit = _CIRCUIT_KEY_CACHE.get(name)
        if hit is not None:
            return hit
        srs = system_srs()
        witness, statement = circuit.dummy_instance()
        try:
            cs = circuit.synthesize(witness, statement, circuit.get_circuit_layout())
            circ = cs.finalize_for_arithmetization()
        except Exception as e:  # mpc-relation CircuitError
            raise ProverError("Circuit", e) from e
        if circ.n + 3 > len(srs.powers_of_g):
            raise ProverError("Plonk", f"circuit {name} needs {circ.n + 3} SRS powers, {len(srs.powers_of_g)} loaded")
        try:
            if getattr(circuit, "prove_from_witness", False):
                pk = PlonkKzgSnark.preprocess_wiring(srs.ctx, srs.powers_of_g, circ.log_n, circ.num_inputs, circ.selectors,
                                                     circ.wire_vars, circ.num_vars, circ.k)
            else:
                pk = PlonkKzgSnark.preprocess(srs.ctx, srs.powers_of_g, circ.log_n, circ.num_inputs, circ.selectors, circ.perm,
                                              circ.k)
        except _lib.B200Error as e:
            raise ProverError("Plonk", e) from e
        pair = (pk, VerifyingKey.from_proving_key(pk, srs.g2_h, srs.g2_tau_h))
        _CIRCUIT_STRUCTURE[name] = int(getattr(circ, "structure_digest", 0) or 0)
        _CIRCUIT_KEY_CACHE[name] = pair
        return pair


class SingleProverCircuit:
    """traits.rs:868-1020.  Subclasses give `name()`, `synthesize`, `statement_scalars`, `dummy_instance` and, when they
    take part in proof linking, `proof_linking_groups()` / `generate_layout`."""

    # Opt-in: the key is built from the circuit's wiring (`preprocess_wiring`) and every proof is made from the witness
    # vector (`prove_witness`): the host never builds the 5 x n value table.  The constraint system's
    # `finalize_for_arithmetization` must then give `wire_vars` / `witness` and take `witness_only=True`.
    prove_from_witness = False

    # ---- what a circuit provides --------------------------------------------------------------------------
    @classmethod
    def name(cls) -> str:
        raise NotImplementedError

    @classmethod
    def synthesize(cls, witness, statement, layout):
        """`PlonkCircuit::new_turbo_plonk()` + link groups of `layout` + `create_witness` / `create_public_var` +
        `apply_constraints` (traits.rs:976-990): returns the constraint system, not yet finalized."""
        raise NotImplementedError

    @classmethod
    def statement_scalars(cls, statement) -> np.ndarray:
        """`statement.to_scalars()` as (num_inputs, 4) Montgomery limbs (traits.rs:1008)."""
        raise NotImplementedError

    @classmethod
    def dummy_instance(cls):
        """(witness, statement) of the circuit's topology for key set-up (the reference uses zeroed scalars)."""
        raise NotImplementedError

    @classmethod
    def proof_linking_groups(cls):
        """[(group id, GroupLayout or None)] — none by default (traits.rs:903-905)."""
        return []

    @classmethod
    def generate_layout(cls):
        """Layout of the link groups (`cs.generate_layout()`, traits.rs:942); None without link groups."""
        return None

    # ---- keys -----------------------------------------------------------------------------------------------
    @classmethod
    def proving_key(cls) -> ProvingKey:
        return setup_preprocessed_keys(cls)[0]

    @classmethod
    def verifying_key(cls) -> VerifyingKey:
        return setup_preprocessed_keys(cls)[1]

    @classmethod
    def get_circuit_layout(cls):
        """traits.rs:914-946: computed once per circuit name."""
        name = cls.name()
        with _KEY_LOCK:
            if name not in _CIRCUIT_LAYOUT_CACHE:
                _CIRCUIT_LAYOUT_CACHE[name] = cls.generate_layout()
            return _CIRCUIT_LAYOUT_CACHE[name]

    # ---- prove / verify ---------------------------------------------------------------------------------------
    @classmethod
    def prove(cls, witness, statement, rng=None) -> PlonkProof:
        return cls.prove_with_link_hint(witness, statement, rng)[0]

    @classmethod
    def prove_with_link_hint(cls, witness, statement, rng=None) -> Tuple[PlonkProof, ProofLinkingHint]:
        pk, circ = cls._arithmetize(witness, statement)
        srs = system_srs()
        try:
            if cls.prove_from_witness:
                if srs.pool is None:
                    return PlonkKzgSnark.prove_witness(srs.ctx, pk, circ.witness, draw_blinders(rng))[:2]
                proof, link, _ = srs.pool.wait(srs.pool.submit_prove_witness(pk, circ.witness, draw_blinders(rng),
                                                                             with_link_poly=True))
                return proof, LinkingHint(linking_wire_poly=link,
                                          linking_wire_comm=np.array(proof.wires_poly_comms[0], dtype=np.uint64))
            if srs.pool is None:
                return PlonkKzgSnark.prove_with_link_hint(srs.ctx, pk, circ.wires, circ.pub_inputs, draw_blinders(rng))
            wires = np.ascontiguousarray(circ.wires, dtype=np.uint64)
            tk = srs.pool.submit_prove(pk, wires.ctypes.data, circ.pub_inputs, draw_blinders(rng), with_link_poly=True,
                                       keep=wires)
            proof, link = srs.pool.wait(tk)
            return proof, LinkingHint(linking_wire_poly=link,
                                      linking_wire_comm=np.array(proof.wires_poly_comms[0], dtype=np.uint64))
        except _lib.B200Error as e:  # WrongQuotientPolyDegree et al.
            raise ProverError("Plonk", e) from e

    @classmethod
    def prove_settlement(cls, witness, statement, hints, rng=None, pool=None, srs_bases=None, urgent=False):
        """A settlement arm of `NativeProofManager::handle_proof_job` (native_proof_manager.rs:514-660) in ONE call:
        `singleprover_prove_with_hint` of this statement, then `link_proofs(hint, &settlement_hint, &layout)` for every
        (stored hint, link group id) in `hints` (validity hint first, intent_and_balance.rs:57-72), the group layouts
        taken from `get_circuit_layout()`.  One settlement job on `pool` (default: the system SRS's pool), else one call
        on the SRS context; `srs_bases` defaults to the system SRS.  The proof and link proofs equal
        `prove_with_link_hint` + `link_proofs` with the same rng.  Returns (proof, [link proofs]); an unsatisfied witness
        or a hint that differs from the statement on its group (a stale hint) raises ProverError("Plonk") naming it.
        `urgent`: on a pool, expedite the job right after submit (`ProverPool.expedite`), so that it overtakes the
        queued proofs and runs on an express worker when the pool has one; the bytes do not change."""
        return settlement_result(hints, *cls.prove_settlement_statuses(witness, statement, hints, rng, pool, srs_bases,
                                                                       urgent))

    @classmethod
    def prove_settlement_statuses(cls, witness, statement, hints, rng=None, pool=None, srs_bases=None, urgent=False):
        """`prove_settlement` without the raising: (proof, link proofs, statuses), statuses[0] the proof's and
        statuses[1 + i] hint i's (0, or B200_ERR_UNSATISFIED)."""
        pk, circ = cls._arithmetize(witness, statement)
        layouts = cls.get_circuit_layout()
        links = [(h, GroupLayout(layouts[g].alignment, layouts[g].offset, layouts[g].size)) for h, g in hints]
        srs = system_srs()
        pool = srs.pool if pool is None else pool
        bases = srs_bases or srs.powers_of_g
        blinders = draw_blinders(rng)
        try:
            if pool is not None:
                tk = (pool.submit_settlement_witness(bases, pk, circ.witness, blinders, links) if cls.prove_from_witness
                      else pool.submit_settlement(bases, pk, circ.wires, circ.pub_inputs, blinders, links))
                res = pool.wait(_expedited(pool, tk, urgent))
            elif cls.prove_from_witness:
                res = PlonkKzgSnark.prove_settlement_witness(srs.ctx, bases, pk, circ.witness, blinders, links)
            else:
                res = PlonkKzgSnark.prove_settlement(srs.ctx, bases, pk, circ.wires, circ.pub_inputs, blinders, links)
        except _lib.B200Error as e:
            raise ProverError("Plonk", e) from e
        return res[:3]

    @classmethod
    def prove_batch_with_link_hint(cls, instances, rng=None) -> List[Tuple[PlonkProof, ProofLinkingHint]]:
        """Many (witness, statement) pairs of this circuit: each is synthesised on the host, then ONE batch call
        (`PlonkKzgSnark.prove_batch`, or one pool job when the SRS has a pool) proves them all.  Raises ProverError naming
        the indices whose witness does not satisfy the circuit."""
        instances = list(instances)
        if not instances:
            return []
        arith = [cls._arithmetize(w, s) for w, s in instances]
        pk = arith[0][0]
        blinders = [draw_blinders(rng) for _ in arith]
        srs = system_srs()
        if not cls.prove_from_witness:
            wires = [np.ascontiguousarray(c.wires, dtype=np.uint64) for _, c in arith]
            pis = [c.pub_inputs for _, c in arith]
        try:
            if cls.prove_from_witness:  # one batch call on the SRS context (the pool has no witness batch job)
                proofs, hints, statuses, _ = PlonkKzgSnark.prove_witness_batch(srs.ctx, pk, [c.witness for _, c in arith],
                                                                               blinders, link_hints=True)
            elif srs.pool is None:
                proofs, hints, statuses = PlonkKzgSnark.prove_batch(srs.ctx, pk, wires, pis, blinders, link_hints=True)
            else:
                tk = srs.pool.submit_prove_batch(pk, wires, pis, blinders, link_hints=True)
                proofs, hints, statuses = srs.pool.wait(tk)
        except _lib.B200Error as e:
            raise ProverError("Plonk", e) from e
        bad = [i for i, st in enumerate(statuses) if st != _lib.B200_OK]
        if bad:
            raise ProverError("Plonk", f"WrongQuotientPolyDegree at indices {bad}")
        return list(zip(proofs, hints))

    @classmethod
    def _arithmetize(cls, witness, statement):
        """The proving key and the witness's arithmetized tables (synthesis on the host), shape-checked against the key."""
        pk = cls.proving_key()
        keyed = _CIRCUIT_STRUCTURE.get(cls.name(), 0)
        try:
            cs = cls.synthesize(witness, statement, cls.get_circuit_layout())
            # the key holds the witness-independent structure; per proof only the value tables are arithmetized
            # (SURVEY 8(f) f4), with a fingerprint of the structure to compare against the key's
            try:
                if cls.prove_from_witness:
                    circ = cs.finalize_for_arithmetization(witness_only=True)
                else:
                    circ = cs.finalize_for_arithmetization(wires_only=True) if keyed else cs.finalize_for_arithmetization()
            except TypeError:  # a constraint system without the wires-only form
                circ = cs.finalize_for_arithmetization()
        except ProverError:
            raise
        except Exception as e:
            raise ProverError("Circuit", e) from e
        if circ.log_n != pk.log_n or circ.num_inputs != pk.num_inputs:
            raise ProverError("Plonk", f"{cls.name()}: instance shape differs from the preprocessed key")
        if keyed and getattr(circ, "structure_digest", 0) and circ.structure_digest != keyed:
            raise ProverError("Circuit", f"{cls.name()}: the instance's gates / wiring differ from the circuit its key was "
                                         "preprocessed from (synthesis must be witness-independent)")
        return pk, circ

    @classmethod
    def verify(cls, statement, proof: PlonkProof) -> None:
        vk = cls.verifying_key()
        try:
            ok = PlonkKzgSnark.verify(vk, cls.statement_scalars(statement), proof)
        except _lib.B200Error as e:
            raise VerifierError(f"Plonk({e})") from e
        if not ok:
            raise VerifierError("Plonk(WrongProof)")


# ---- circuits-core/src/lib.rs:112-142 ------------------------------------------------------------------------------
def singleprover_prove(circuit: type, witness, statement, rng=None) -> PlonkProof:
    return circuit.prove(witness, statement, rng)


def singleprover_prove_with_hint(circuit: type, witness, statement, rng=None) -> Tuple[PlonkProof, ProofLinkingHint]:
    return circuit.prove_with_link_hint(witness, statement, rng)


def settlement_result(hints, proof, link_proofs, statuses):
    """(proof, link proofs) of a settlement whose statuses are all B200_OK; else ProverError("Plonk") naming the failure:
    an unsatisfied settlement witness, or the hints that differ from the statement on their link group (stale hints)."""
    if statuses[0] != _lib.B200_OK:
        raise ProverError("Plonk", "WrongQuotientPolyDegree: the settlement witness does not satisfy the circuit")
    stale = [f"hint {i} (group {hints[i][1]})" for i in range(len(hints)) if statuses[1 + i] != _lib.B200_OK]
    if stale:
        raise ProverError("Plonk", f"{', '.join(stale)}: differs from the settlement on its link group (a stale hint)")
    return proof, link_proofs


def singleprover_prove_settlement(circuit: type, witness, statement, hints, rng=None):
    """`SingleProverCircuit.prove_settlement`: (proof, [link proofs]) of a settlement against its stored hints."""
    return circuit.prove_settlement(witness, statement, hints, rng)


def singleprover_prove_batch(circuit: type, instances, rng=None) -> List[PlonkProof]:
    """`singleprover_prove` for many (witness, statement) pairs of one circuit in ONE batch call on the device; raises
    ProverError naming the indices whose witness does not satisfy the circuit."""
    return [p for p, _ in circuit.prove_batch_with_link_hint(instances, rng)]


def singleprover_prove_batch_with_hint(circuit: type, instances, rng=None) -> List[Tuple[PlonkProof, ProofLinkingHint]]:
    return circuit.prove_batch_with_link_hint(instances, rng)


def verify_singleprover_proof(circuit: type, statement, proof: PlonkProof) -> None:
    circuit.verify(statement, proof)


def _expedited(jobs, ticket: int, urgent: bool) -> int:
    """The ticket, expedited on its pool or box first when `urgent` (the job overtakes the queued ones)."""
    if urgent:
        jobs.expedite(ticket)
    return ticket


def batch_verify_singleprover_proofs(items, pool=None, box=None, urgent=False) -> None:
    """`verify_singleprover_proof` for many (circuit, statement, proof) triples at once: one batch check with ONE
    pairing on the `SYSTEM_SRS` context's device (`PlonkKzgSnark.batch_verify`), or, given a `ProverPool` as `pool` or a
    `ProverBox` as `box`, the same check as one verification job on it (`submit_verify(..., combined=True)`), beside the
    proofs it is making; `urgent` expedites that job right after submit.  Raises VerifierError naming the indices of the
    proofs that fail."""
    items = list(items)
    if not items:
        return
    if pool is not None and box is not None:
        raise ValueError("batch_verify_singleprover_proofs: pass a pool or a box, not both")
    vks = [c.verifying_key() for c, _, _ in items]
    pis = [c.statement_scalars(s) for c, s, _ in items]
    proofs = [p for _, _, p in items]
    try:
        if pool is not None or box is not None:
            jobs = pool if pool is not None else box
            _, verdicts = jobs.wait(_expedited(jobs, jobs.submit_verify(vks, pis, proofs, combined=True), urgent))
        else:
            _, verdicts = PlonkKzgSnark.batch_verify(system_srs().ctx, vks, pis, proofs)
    except _lib.B200Error as e:
        raise VerifierError(f"Plonk({e})") from e
    bad = [i for i, ok in enumerate(verdicts) if not ok]
    if bad:
        raise VerifierError(f"Plonk(WrongProof) at indices {bad}")


def singleprover_prove_and_verify(circuit: type, witness, statement, rng=None) -> None:
    proof = circuit.prove(witness, statement, rng)
    try:
        circuit.verify(statement, proof)
    except VerifierError as e:
        raise ProverError("Verification", e) from e


# ---- circuit-types/src/traits.rs:1103-1154, circuits-core/src/lib.rs:145-177 -------------------------------------------
class MultiProverCircuit:
    """`MultiProverCircuit`: the collaborative counterpart of a `SingleProverCircuit` (the reference pairs them: a
    statement's `MultiProverCircuit` impl names its `BaseCircuit`, and the opened proof verifies under the SAME keys,
    traits.rs:1103-1154).  Subclasses set `BaseCircuit`.

    `prove_with_link_hint(witness_shares, statement)`: every party's share of the 5 x n wire table (and of the 17
    blinders) goes into `collaborative.MultiproverPlonkKzgSnark` on the device; what comes back is the OPENED proof and
    hint (`open_authenticated` in `multiprover_prove_and_verify`, lib.rs:166-177).  Producing the wire-table shares —
    running the constraint system on shared values (`MpcPlonkCircuit`) — is the callers' side, like single-prover
    synthesis; `share_witness_table` stands in for it where a test or an example starts from a clear witness."""
    BaseCircuit: type = None

    @classmethod
    def share_witness_table(cls, witness, statement, parties: int = 2, seed: int = 0):
        from .collaborative import share_table
        base = cls.BaseCircuit
        circ = base.synthesize(witness, statement, base.get_circuit_layout()).finalize_for_arithmetization()
        return circ, share_table(np.asarray(circ.wires, dtype=np.uint64).reshape(-1, 4), parties, seed)

    @classmethod
    def prove_with_link_hint(cls, circ, wire_shares, blinder_shares=None, rng=None):
        """`circ`: the finalized public circuit structure (selectors, permutation, public inputs); `wire_shares[p]`:
        party p's share of its wire table.  Returns (PlonkProof, ProofLinkingHint) — opened."""
        from . import collaborative as co
        srs = system_srs()
        be = co.DeviceBackend(srs.ctx, srs.powers_of_g)
        parties = len(wire_shares)
        if blinder_shares is None:
            blinder_shares = co.share_table(draw_blinders(rng), parties, seed=int.from_bytes(os.urandom(8), "little"))
        try:
            cpk = co.CollaborativeProvingKey.build(be, circ.log_n, circ.num_inputs, circ.selectors, circ.perm, circ.k)
            proof, hint, _ = co.MultiproverPlonkKzgSnark.prove_with_link_hint(be, cpk, wire_shares, circ.pub_inputs, blinder_shares)
        except _lib.B200Error as e:
            raise ProverError("Plonk", e) from e
        return proof, hint

    @classmethod
    def verify(cls, statement, proof: PlonkProof) -> None:
        cls.BaseCircuit.verify(statement, proof)


def multiprover_prove_with_hint(circuit: type, circ, wire_shares, blinder_shares=None, rng=None):
    return circuit.prove_with_link_hint(circ, wire_shares, blinder_shares, rng)


def multiprover_prove_and_verify(circuit: type, witness, statement, parties: int = 2, rng=None) -> None:
    """lib.rs:166-177: prove collaboratively, open, verify under the base circuit's verifying key."""
    circ, shares = circuit.share_witness_table(witness, statement, parties)
    proof, _ = circuit.prove_with_link_hint(circ, shares, rng=rng)
    try:
        circuit.verify(statement, proof)
    except VerifierError as e:
        raise ProverError("Verification", e) from e
