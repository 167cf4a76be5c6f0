"""TEST INFRASTRUCTURE — ctypes loader for oracle/_build/liboracle.so (the C restatement).
Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may
import this.  Arrays are numpy uint64 with trailing dimension 4 (field element, LE limbs) or
8 (G1 affine x||y, Montgomery)."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "_build", "liboracle.so")

FR, FQ = 0, 1


def build(force: bool = False) -> str:
    srcs = [os.path.join(_HERE, f) for f in os.listdir(_HERE) if f.endswith((".c", ".h"))]
    stale = (not os.path.exists(_SO)) or any(os.path.getmtime(s) > os.path.getmtime(_SO) for s in srcs)
    if force or stale:
        subprocess.check_call(["make", "-C", _HERE, "-s"])
    return _SO


_lib = None


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(_SO):
            build()
        # idle OpenMP workers must sleep, not spin: the GPU box's host CPUs are shared
        os.environ.setdefault("OMP_WAIT_POLICY", "passive")
        _lib = C.CDLL(_SO)
        _lib.orc_msm_window_bits.restype = C.c_int
        _lib.orc_msm_window_bits.argtypes = [C.c_size_t]
        _lib.orc_num_threads.restype = C.c_int
        _lib.orc_g1_on_curve.restype = C.c_int
    return _lib


def _p(a: np.ndarray):
    assert a.dtype == np.uint64 and a.flags["C_CONTIGUOUS"]
    return a.ctypes.data_as(C.c_void_p)


def int_to_limbs(v: int) -> np.ndarray:
    return np.array([(v >> (64 * i)) & 0xFFFFFFFFFFFFFFFF for i in range(4)], dtype=np.uint64)


def limbs_to_int(a) -> int:
    a = np.asarray(a, dtype=np.uint64).reshape(-1)
    return sum(int(a[i]) << (64 * i) for i in range(len(a)))


def ints_to_array(vals) -> np.ndarray:
    out = np.zeros((len(vals), 4), dtype=np.uint64)
    for i, v in enumerate(vals):
        out[i] = int_to_limbs(v)
    return out


def array_to_ints(a: np.ndarray):
    a = np.asarray(a, dtype=np.uint64).reshape(-1, 4)
    return [limbs_to_int(r) for r in a]


def fp_binop(name: str, which: int, a: np.ndarray, b: np.ndarray) -> np.ndarray:
    out = np.zeros(4, dtype=np.uint64)
    getattr(lib(), name)(C.c_int(which), _p(np.ascontiguousarray(a)), _p(np.ascontiguousarray(b)), _p(out))
    return out


def fp_unop(name: str, which: int, a: np.ndarray) -> np.ndarray:
    out = np.zeros(4, dtype=np.uint64)
    getattr(lib(), name)(C.c_int(which), _p(np.ascontiguousarray(a)), _p(out))
    return out


def array_from_mont(which: int, a: np.ndarray) -> np.ndarray:
    a = np.ascontiguousarray(a, dtype=np.uint64)
    out = np.empty_like(a)
    lib().orc_fp_array_from_mont(C.c_int(which), _p(a), C.c_size_t(a.size // 4), _p(out))
    return out


def array_to_mont(which: int, a: np.ndarray) -> np.ndarray:
    a = np.ascontiguousarray(a, dtype=np.uint64)
    out = np.empty_like(a)
    lib().orc_fp_array_to_mont(C.c_int(which), _p(a), C.c_size_t(a.size // 4), _p(out))
    return out


def splitmix_fr(seed: int, n: int, montgomery: bool, first: int = 0) -> np.ndarray:
    out = np.empty((n, 4), dtype=np.uint64)
    lib().orc_splitmix_fr(C.c_uint64(seed), C.c_size_t(first), C.c_size_t(n), C.c_int(int(montgomery)), _p(out))
    return out


def known_dlog_bases(seed: int, n: int, first: int = 0) -> np.ndarray:
    out = np.empty((n, 8), dtype=np.uint64)
    lib().orc_g1_known_dlog_bases(C.c_uint64(seed), C.c_size_t(first), C.c_size_t(n), _p(out))
    return out


def fr_dot(seed_a: int, seed_b: int, n: int, first_a: int = 0, first_b: int = 0) -> int:
    """sum_i a_i b_i mod r over i < n, a = splitmix_fr(seed_a, first=first_a), b = splitmix_fr(seed_b, first=first_b):
    the discrete log of an MSM of known-dlog bases with SplitMix scalars, computed without materialising either vector."""
    out = np.zeros(4, dtype=np.uint64)
    lib().orc_fr_dot(C.c_uint64(seed_a), C.c_size_t(first_a), C.c_uint64(seed_b), C.c_size_t(first_b), C.c_size_t(n),
                     _p(out))
    return limbs_to_int(out)


def g1_on_curve(xy: np.ndarray) -> bool:
    return bool(lib().orc_g1_on_curve(_p(np.ascontiguousarray(xy, dtype=np.uint64))))


def g1_add(a, a_inf, b, b_inf):
    out = np.zeros(8, dtype=np.uint64)
    inf = C.c_int(0)
    lib().orc_g1_add(_p(np.ascontiguousarray(a)), C.c_int(int(a_inf)), _p(np.ascontiguousarray(b)),
                     C.c_int(int(b_inf)), _p(out), C.byref(inf))
    return out, bool(inf.value)


def g1_mul(p, p_inf, k_canon):
    out = np.zeros(8, dtype=np.uint64)
    inf = C.c_int(0)
    lib().orc_g1_mul(_p(np.ascontiguousarray(p)), C.c_int(int(p_inf)), _p(np.ascontiguousarray(k_canon)),
                     _p(out), C.byref(inf))
    return out, bool(inf.value)


def msm(bases: np.ndarray, scalars_canon: np.ndarray, naive: bool = False):
    bases = np.ascontiguousarray(bases, dtype=np.uint64)
    scalars_canon = np.ascontiguousarray(scalars_canon, dtype=np.uint64)
    n = min(bases.size // 8, scalars_canon.size // 4)
    out = np.zeros(8, dtype=np.uint64)
    inf = C.c_int(0)
    fn = lib().orc_msm_naive if naive else lib().orc_msm
    fn(_p(bases), _p(scalars_canon), C.c_size_t(n), _p(out), C.byref(inf))
    return out, bool(inf.value)


def msm_window_bits(n: int) -> int:
    return lib().orc_msm_window_bits(n)


def ntt(data: np.ndarray, inverse: bool = False, coset: bool = False) -> np.ndarray:
    """Returns a transformed copy (Montgomery in, Montgomery out, natural order)."""
    out = np.array(data, dtype=np.uint64, copy=True, order="C")
    n = out.size // 4
    log_n = n.bit_length() - 1
    assert 1 << log_n == n
    lib().orc_ntt(_p(out), C.c_uint(log_n), C.c_int(int(inverse)), C.c_int(int(coset)))
    return out


def domain_generator(log_n: int) -> np.ndarray:
    out = np.zeros(4, dtype=np.uint64)
    lib().orc_domain_generator(C.c_uint(log_n), _p(out))
    return out


def num_threads() -> int:
    return lib().orc_num_threads()


def set_num_threads(n: int) -> None:
    lib().orc_set_num_threads(C.c_int(n))


def autotune_threads(candidates=None) -> int:
    """Pick the OpenMP thread count that runs a small MSM + NTT fastest on this host (on a shared
    box "all logical CPUs" can be far slower than a subset) and keep it.  Returns the choice."""
    import time
    ncpu = len(os.sched_getaffinity(0)) if hasattr(os, "sched_getaffinity") else (os.cpu_count() or 1)
    if candidates is None:
        candidates = sorted({c for c in (ncpu, ncpu // 2, 64, 32, 16, 8) if 1 <= c <= ncpu}, reverse=True)
    bases = known_dlog_bases(1, 1 << 13)
    sc = splitmix_fr(2, 1 << 13, False)
    x = splitmix_fr(3, 1 << 16, True)
    best, best_t = candidates[-1], float("inf")
    for c in candidates:
        set_num_threads(c)
        msm(bases, sc)
        t = time.perf_counter()
        for _ in range(3):
            msm(bases, sc)
            ntt(x)
        dt = time.perf_counter() - t
        if dt < best_t:
            best, best_t = c, dt
    set_num_threads(best)
    return best


# ---------------------------------------------------------------------------------------------
# Poseidon2, t = 3 (poseidon2_oracle.c).  Arrays are Montgomery limbs, like the device calls'.
# ---------------------------------------------------------------------------------------------
POSEIDON2_FIXTURE = os.path.join(os.path.dirname(_HERE), "tests", "golden", "poseidon2.json")
_p2_rc = None


def poseidon2_round_constants():
    """(full (24, 4), partial (56, 4)) Montgomery round constants, read from the fixture (not from the product)."""
    global _p2_rc
    if _p2_rc is None:
        import json
        with open(POSEIDON2_FIXTURE) as f:
            d = json.load(f)
        full = ints_to_array([int(v, 16) for v in d["full_round_constants"]])
        partial = ints_to_array([int(v, 16) for v in d["partial_round_constants"]])
        assert full.shape == (24, 4) and partial.shape == (56, 4)
        _p2_rc = (array_to_mont(FR, full), array_to_mont(FR, partial))
    return _p2_rc


def poseidon2_permute_batch(states: np.ndarray) -> np.ndarray:
    """(batch, 3, 4) states -> permuted copy."""
    out = np.array(states, dtype=np.uint64, copy=True, order="C").reshape(-1, 3, 4)
    full, partial = poseidon2_round_constants()
    lib().orc_poseidon2_permute_batch(_p(out), C.c_size_t(out.shape[0]), _p(full), _p(partial))
    return out


def poseidon2_hash_batch(values: np.ndarray) -> np.ndarray:
    """(batch, len, 4) -> (batch, 4): one sponge hash per row (len may be 0)."""
    v = np.ascontiguousarray(values, dtype=np.uint64)
    batch, ln = v.shape[0], v.shape[1]
    out = np.zeros((batch, 4), dtype=np.uint64)
    if batch == 0:
        return out
    full, partial = poseidon2_round_constants()
    lib().orc_poseidon2_hash_batch(_p(v) if v.size else None, C.c_size_t(batch), C.c_size_t(ln), _p(full), _p(partial),
                                   _p(out))
    return out


def poseidon2_merkle_roots(leaves: np.ndarray, sisters: np.ndarray, is_right: np.ndarray) -> np.ndarray:
    """leaves (batch, 4), sisters (batch, height, 4), is_right (batch, height) -> (batch, 4): per level one batched
    two-to-one hash, H(sister, cur) where is_right != 0, else H(cur, sister)."""
    cur = np.ascontiguousarray(leaves, dtype=np.uint64).reshape(-1, 4)
    sis = np.asarray(sisters, dtype=np.uint64).reshape(cur.shape[0], -1, 4)
    right = np.asarray(is_right).reshape(cur.shape[0], sis.shape[1]) != 0
    for lvl in range(sis.shape[1]):
        r = right[:, lvl, None]
        cur = poseidon2_hash_batch(np.stack([np.where(r, sis[:, lvl], cur), np.where(r, cur, sis[:, lvl])], axis=1))
    return cur


def poseidon2_csprng(seeds: np.ndarray, first_index, count: int) -> np.ndarray:
    """seeds (batch, 4), first_index (batch,) -> (batch, count, 4): value j of stream s is H(seed_s, first_s + j)."""
    sd = np.ascontiguousarray(seeds, dtype=np.uint64).reshape(-1, 4)
    first = [int(f) for f in first_index]
    assert len(first) == sd.shape[0] and all(0 <= f and f + count <= 1 << 64 for f in first)
    idx = np.zeros((sd.shape[0], count, 4), dtype=np.uint64)
    idx[:, :, 0] = np.array(first, dtype=np.uint64)[:, None] + np.arange(count, dtype=np.uint64)[None, :]
    pairs = np.stack([np.repeat(sd[:, None], count, axis=1), array_to_mont(FR, idx)], axis=2)
    return poseidon2_hash_batch(pairs.reshape(-1, 2, 4)).reshape(sd.shape[0], count, 4)


# ---------------------------------------------------------------------------------------------
# TurboPlonk prover / verifier restatement (plonk_oracle.c)
# ---------------------------------------------------------------------------------------------
class PlonkProof(C.Structure):
    """orc_plonk_proof — field order mirrors PlonkProofDef (plonk_proof_def.rs:197-222)."""
    _fields_ = [
        ("wires_poly_comms", (C.c_uint64 * 8) * 5),
        ("prod_perm_poly_comm", C.c_uint64 * 8),
        ("split_quot_poly_comms", (C.c_uint64 * 8) * 5),
        ("opening_proof", C.c_uint64 * 8),
        ("shifted_opening_proof", C.c_uint64 * 8),
        ("wires_evals", (C.c_uint64 * 4) * 5),
        ("wire_sigma_evals", (C.c_uint64 * 4) * 4),
        ("perm_next_eval", C.c_uint64 * 4),
    ]

    def to_array(self) -> np.ndarray:
        return np.frombuffer(bytes(self), dtype=np.uint64).copy()


class PlonkChallenges(C.Structure):
    _fields_ = [(n, C.c_uint64 * 4) for n in ("beta", "gamma", "alpha", "zeta", "v", "u")]


def keccak256(data: bytes) -> bytes:
    out = (C.c_uint8 * 32)()
    lib().orc_keccak256(data, C.c_size_t(len(data)), out)
    return bytes(out)


def srs_from_tau(tau_mont: np.ndarray, n: int) -> np.ndarray:
    out = np.empty((n, 8), dtype=np.uint64)
    lib().orc_srs_from_tau(_p(np.ascontiguousarray(tau_mont, dtype=np.uint64)), C.c_size_t(n), _p(out))
    return out


def plonk_preprocess(log_n, selectors, perm, k, srs):
    n = 1 << log_n
    selectors = np.ascontiguousarray(selectors, dtype=np.uint64)
    perm = np.ascontiguousarray(perm, dtype=np.uint64)
    k = np.ascontiguousarray(k, dtype=np.uint64)
    srs = np.ascontiguousarray(srs, dtype=np.uint64)
    sel_c = np.empty((13, n, 4), dtype=np.uint64)
    sig_c = np.empty((5, n, 4), dtype=np.uint64)
    sel_comms = np.empty((13, 8), dtype=np.uint64)
    sig_comms = np.empty((5, 8), dtype=np.uint64)
    rc = lib().orc_plonk_preprocess(C.c_uint(log_n), _p(selectors), _p(perm), _p(k), _p(srs), _p(sel_c), _p(sig_c),
                                    _p(sel_comms), _p(sig_comms))
    assert rc == 0
    return {"selector_coeffs": sel_c, "sigma_coeffs": sig_c, "selector_comms": sel_comms, "sigma_comms": sig_comms}


def plonk_prove(log_n, num_inputs, k, pk, wires, pub_inputs, blinders, srs, want_link_poly=False):
    n = 1 << log_n
    proof, ch = PlonkProof(), PlonkChallenges()
    link = np.zeros((n + 2, 4), dtype=np.uint64) if want_link_poly else None
    lib().orc_plonk_prove.restype = C.c_int
    rc = lib().orc_plonk_prove(
        C.c_uint(log_n), C.c_size_t(num_inputs), _p(np.ascontiguousarray(k, dtype=np.uint64)),
        _p(pk["selector_coeffs"]), _p(pk["sigma_coeffs"]), _p(pk["selector_comms"]), _p(pk["sigma_comms"]),
        _p(np.ascontiguousarray(wires, dtype=np.uint64)), _p(np.ascontiguousarray(pub_inputs, dtype=np.uint64)),
        _p(np.ascontiguousarray(blinders, dtype=np.uint64)), _p(np.ascontiguousarray(srs, dtype=np.uint64)),
        C.byref(proof), C.byref(ch), _p(link) if link is not None else None)
    return rc, proof, ch, link


def plonk_verify_known_tau(log_n, num_inputs, k, pk, pub_inputs, proof: PlonkProof, tau_mont) -> bool:
    lib().orc_plonk_verify_known_tau.restype = C.c_int
    return bool(lib().orc_plonk_verify_known_tau(
        C.c_uint(log_n), C.c_size_t(num_inputs), _p(np.ascontiguousarray(k, dtype=np.uint64)),
        _p(pk["selector_comms"]), _p(pk["sigma_comms"]), _p(np.ascontiguousarray(pub_inputs, dtype=np.uint64)),
        C.byref(proof), _p(np.ascontiguousarray(tau_mont, dtype=np.uint64))))


class LinkProof(C.Structure):
    """orc_link_proof / mpc-plonk `LinkingProof { quotient_commitment, opening_proof }`."""
    _fields_ = [("quotient_commitment", C.c_uint64 * 8), ("opening_proof", C.c_uint64 * 8)]

    def to_array(self) -> np.ndarray:
        return np.frombuffer(bytes(self), dtype=np.uint64).copy()


def plonk_link(a1, a2, comm1, comm2, alignment, offset, size, srs):
    a1 = np.ascontiguousarray(a1, dtype=np.uint64).reshape(-1, 4)
    a2 = np.ascontiguousarray(a2, dtype=np.uint64).reshape(-1, 4)
    proof = LinkProof()
    eta = np.zeros(4, dtype=np.uint64)
    lib().orc_plonk_link.restype = C.c_int
    rc = lib().orc_plonk_link(_p(a1), C.c_size_t(a1.shape[0]), _p(a2), C.c_size_t(a2.shape[0]),
                              _p(np.ascontiguousarray(comm1, dtype=np.uint64)), _p(np.ascontiguousarray(comm2, dtype=np.uint64)),
                              C.c_uint(alignment), C.c_size_t(offset), C.c_size_t(size),
                              _p(np.ascontiguousarray(srs, dtype=np.uint64)), C.byref(proof), _p(eta))
    return rc, proof, eta


def plonk_link_verify_known_tau(comm1, comm2, alignment, offset, size, proof: LinkProof, tau_mont) -> bool:
    lib().orc_plonk_link_verify_known_tau.restype = C.c_int
    return bool(lib().orc_plonk_link_verify_known_tau(
        _p(np.ascontiguousarray(comm1, dtype=np.uint64)), _p(np.ascontiguousarray(comm2, dtype=np.uint64)),
        C.c_uint(alignment), C.c_size_t(offset), C.c_size_t(size), C.byref(proof),
        _p(np.ascontiguousarray(tau_mont, dtype=np.uint64))))


def plonk_verify_operands(log_n, num_inputs, k, pk, pub_inputs, proof: PlonkProof):
    """G1 operands (A, B) of the pairing check e(A, [tau]_2) == e(B, [1]_2); each is an (x||y Montgomery, is_identity) pair."""
    a, b = np.zeros(8, dtype=np.uint64), np.zeros(8, dtype=np.uint64)
    ai, bi = C.c_int(0), C.c_int(0)
    lib().orc_plonk_verify_operands(
        C.c_uint(log_n), C.c_size_t(num_inputs), _p(np.ascontiguousarray(k, dtype=np.uint64)),
        _p(pk["selector_comms"]), _p(pk["sigma_comms"]), _p(np.ascontiguousarray(pub_inputs, dtype=np.uint64)),
        C.byref(proof), _p(a), C.byref(ai), _p(b), C.byref(bi))
    return (a, bool(ai.value)), (b, bool(bi.value))


def plonk_verify_pairing(log_n, num_inputs, k, pk, pub_inputs, proof: PlonkProof, g2_h, g2_tau_h) -> bool:
    """`PlonkKzgSnark::verify` for an SRS with unknown tau: e(A, tau H) * e(-B, H) == 1, with the pairing of
    oracle/bn254_pairing_py.py (g2_h, g2_tau_h as decoded by bn254_pairing_py.decode_g2_mont)."""
    import bn254_pairing_py as pr
    import bn254_py as py
    (a, a_inf), (b, b_inf) = plonk_verify_operands(log_n, num_inputs, k, pk, pub_inputs, proof)
    pa = None if a_inf else py.decode_g1_mont(a.tobytes(), 0)
    pb = None if b_inf else py.g1_neg(py.decode_g1_mont(b.tobytes(), 0))
    return pr.pairing_product_is_one([(pa, g2_tau_h), (pb, g2_h)])
