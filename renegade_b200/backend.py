"""Host-side mirror of the reference's interface for the proving hot path, over the C ABI.

Names follow the Rust surface the reference calls (SURVEY.md §8(a)/(b)):

  parse_ptau_file                      crates/circuits/circuit-types/src/primitives/srs.rs:63-71
  UnivariateUniversalParams            jf-primitives (built at srs.rs:70)
  VariableBaseMSM.msm_bigint           ark-ec 0.4.2 (under UnivariateKzgPCS::commit)
  UnivariateKzgPCS.commit              jf-primitives (reached from traits.rs:850,996)
  Radix2EvaluationDomain               ark-poly 0.4.2 (fft / ifft / coset_fft / coset_ifft)

Field elements are numpy uint64 arrays with a trailing dimension of 4 (little-endian limbs,
Montgomery form unless stated), G1 affine points have a trailing dimension of 8 (x || y).
All arithmetic runs in libb200prover.so on the GPU; nothing here computes on the host.
"""
from __future__ import annotations

import ctypes as C
import functools
from dataclasses import dataclass
from typing import NamedTuple

import numpy as np

from . import _lib

MAX_SRS_POWER = 17
MAX_SRS_DEGREE = (1 << MAX_SRS_POWER) + 2  # srs.rs:44-47


def _ptr(a: np.ndarray):
    assert a.dtype == np.uint64 and a.flags["C_CONTIGUOUS"]
    return a.ctypes.data_as(C.c_void_p)


class Context:
    """One CUDA device + stream + scratch (b200_ctx).  Calls on one context are serialised."""

    def __init__(self, device: int = 0):
        self._lib = _lib.load()
        h = C.c_void_p()
        _lib.check(self._lib.b200_init(device, C.byref(h)))
        self._h = h
        self.device = device

    def close(self):
        if getattr(self, "_h", None):
            self._lib.b200_shutdown(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def use_graphs(self, on: bool = True):
        """Replay the prover's rounds as CUDA graphs from the second proof of a key on (default: on; B200_GRAPHS=0)."""
        _lib.check(self._lib.b200_ctx_use_graphs(self._h, int(on)))

    def kernel_launches(self) -> int:
        """Kernels the library has launched (or replayed inside graphs) in this process so far."""
        return int(self._lib.b200_kernel_launches())

    def graph_launches(self) -> int:
        return int(self._lib.b200_graph_launches())

    # ---- bases / SRS ------------------------------------------------------------------------
    def load_bases(self, points, window_bits: int = 0, check_on_curve: bool = False) -> "Bases":
        """points: (n, 8) uint64 array or bytes of 64-byte records."""
        if isinstance(points, (bytes, bytearray, memoryview)):
            buf = np.frombuffer(bytes(points), dtype=np.uint64).reshape(-1, 8)
        else:
            buf = np.ascontiguousarray(points, dtype=np.uint64).reshape(-1, 8)
        h = C.c_void_p()
        _lib.check(self._lib.b200_bases_load(self._h, _ptr(buf), buf.shape[0], window_bits,
                                             int(check_on_curve), C.byref(h)))
        return Bases(self, h)

    def load_bases_device(self, d_ptr: int, n: int, window_bits: int = 0) -> "Bases":
        h = C.c_void_p()
        _lib.check(self._lib.b200_bases_load_device(self._h, C.c_void_p(d_ptr), n, window_bits, C.byref(h)))
        return Bases(self, h)

    # ---- MSM --------------------------------------------------------------------------------
    def msm(self, bases: "Bases", scalars: np.ndarray, montgomery: bool = False, base_off: int = 0):
        s = np.ascontiguousarray(scalars, dtype=np.uint64).reshape(-1, 4)
        out = np.zeros(8, dtype=np.uint64)
        inf = C.c_int(0)
        _lib.check(self._lib.b200_msm(self._h, bases._h, base_off, _ptr(s), s.shape[0], int(montgomery),
                                      _ptr(out), C.byref(inf)))
        return out, bool(inf.value)

    def msm_device(self, bases: "Bases", d_scalars: int, n: int, montgomery: bool = False, base_off: int = 0):
        out = np.zeros(8, dtype=np.uint64)
        inf = C.c_int(0)
        _lib.check(self._lib.b200_msm_device(self._h, bases._h, base_off, C.c_void_p(d_scalars), n,
                                             int(montgomery), _ptr(out), C.byref(inf)))
        return out, bool(inf.value)

    def msm_timing(self, enable: bool = True) -> dict:
        """Enable device-side phase timing; returns the last MSM's phases in ms."""
        arr = (C.c_float * 4)()
        _lib.check(self._lib.b200_msm_timing(self._h, int(enable), C.byref(arr)))
        return {"total": arr[0], "sort": arr[1], "accumulate": arr[2], "reduce": arr[3]}

    def msm_tuning(self, throughput_mode: bool) -> None:
        """False (default): latency-tuned MSM; True: throughput-tuned (longer per-thread chains in the bucket
        reduction, fewer operations) — same results, for when several MSMs are in flight on the GPU."""
        _lib.check(self._lib.b200_msm_tuning(self._h, int(throughput_mode)))

    def msm_timing_totals(self, reset: bool = False) -> dict:
        """Bucket-accumulation totals since the last reset (timing must be enabled): ms, pairs, launches."""
        arr = (C.c_double * 3)()
        _lib.check(self._lib.b200_msm_timing_totals(self._h, int(reset), C.byref(arr)))
        return {"accumulate_ms": arr[0], "pairs": arr[1], "launches": arr[2]}

    def ntt_last_ms(self) -> float:
        v = C.c_float(0)
        _lib.check(self._lib.b200_ntt_last_ms(self._h, C.byref(v)))
        return v.value

    def g1_sum_affine(self, points: np.ndarray, is_identity=None):
        p = np.ascontiguousarray(points, dtype=np.uint64).reshape(-1, 8)
        flags = None
        if is_identity is not None:
            flags = (C.c_int * p.shape[0])(*[int(bool(x)) for x in is_identity])
        out = np.zeros(8, dtype=np.uint64)
        inf = C.c_int(0)
        _lib.check(self._lib.b200_g1_sum_affine(_ptr(p), flags, p.shape[0], _ptr(out), C.byref(inf)))
        return out, bool(inf.value)

    # ---- NTT --------------------------------------------------------------------------------
    def ntt(self, data: np.ndarray, inverse: bool = False, coset: bool = False) -> np.ndarray:
        out = np.array(data, dtype=np.uint64, copy=True, order="C").reshape(-1, 4)
        n = out.shape[0]
        log_n = n.bit_length() - 1
        if n == 0 or (1 << log_n) != n:
            raise ValueError("domain size must be a power of two")
        _lib.check(self._lib.b200_ntt(self._h, _ptr(out), log_n, int(inverse), int(coset)))
        return out

    def ntt_device(self, d_ptr: int, log_n: int, inverse: bool = False, coset: bool = False,
                   batch: int = 1, stride: int | None = None) -> None:
        stride = (1 << log_n) if stride is None else stride
        _lib.check(self._lib.b200_ntt_device(self._h, C.c_void_p(d_ptr), log_n, int(inverse), int(coset),
                                             batch, stride))

    def domain_generator(self, log_n: int) -> np.ndarray:
        out = np.zeros(4, dtype=np.uint64)
        _lib.check(self._lib.b200_domain_generator(self._h, log_n, _ptr(out)))
        return out

    # ---- synthetic inputs (device) ------------------------------------------------------------
    def splitmix_fr_device(self, seed: int, n: int, d_out: int, montgomery: bool, first: int = 0) -> None:
        _lib.check(self._lib.b200_splitmix_fr_device(self._h, seed, first, n, int(montgomery), C.c_void_p(d_out)))

    def known_dlog_bases_device(self, seed: int, n: int, d_out: int, first: int = 0) -> None:
        _lib.check(self._lib.b200_known_dlog_bases_device(self._h, seed, first, n, C.c_void_p(d_out)))

    # ---- self tests -----------------------------------------------------------------------------
    def selftest_field(self, seed: int, iters: int) -> int:
        bad = C.c_uint64(0)
        _lib.check(self._lib.b200_selftest_field(self._h, seed, iters, C.byref(bad)))
        return bad.value

    def selftest_pairing(self, seed: int, iters: int) -> int:
        """Mismatches between the 16-lane pairing arithmetic and the one-thread pairing functions over `iters` seeded
        operands of every operation (`b200_selftest_pairing`); 0 expected."""
        bad = C.c_uint64(0)
        _lib.check(self._lib.b200_selftest_pairing(self._h, seed, iters, C.byref(bad)))
        return bad.value

    def field_op(self, field: int, op: int, a: np.ndarray, b: np.ndarray) -> np.ndarray:
        a = np.ascontiguousarray(a, dtype=np.uint64).reshape(-1, 4)
        b = np.ascontiguousarray(b, dtype=np.uint64).reshape(-1, 4)
        out = np.zeros_like(a)
        _lib.check(self._lib.b200_field_op(self._h, field, op, _ptr(a), _ptr(b), a.shape[0], _ptr(out)))
        return out


class Bases:
    """Device-resident G1 bases with their precomputed window tables (b200_bases)."""

    def __init__(self, ctx: Context, handle):
        self._ctx = ctx
        self._h = handle

    def __len__(self) -> int:
        return int(self._ctx._lib.b200_bases_len(self._h))

    @property
    def plan(self) -> dict:
        arr = (C.c_int * 4)()
        self._ctx._lib.b200_bases_plan(self._h, C.byref(arr))
        return {"window_bits": arr[0], "digits": arr[1], "physical_windows": arr[2], "tables": arr[3]}

    def free(self):
        if self._h:  # a context that is already gone is passed as NULL (the library allows it)
            self._ctx._lib.b200_bases_free(self._ctx._h, self._h)
        self._h = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


# ---------------------------------------------------------------------------------------------
# Reference-shaped interface
# ---------------------------------------------------------------------------------------------
@dataclass
class UnivariateUniversalParams:
    """jf-primitives `UnivariateUniversalParams<Bn254>` as built at srs.rs:70: the G1 powers
    live on the device; `powers_of_g_host` keeps the raw 64-byte records for inspection.  `h` / `beta_h` are the
    two G2 records of section 3 (16 x uint64 each), None for a truncated file that ends before them."""
    powers_of_g: Bases
    powers_of_g_host: np.ndarray
    h: np.ndarray | None = None
    beta_h: np.ndarray | None = None


def read_ptau_g2(data: bytes):
    """srs.rs:147-157 (`read_ptau_section3`): (h, beta_h), the first two G2 records of section 3, 16 x uint64 each
    (`b200_srs_parse_ptau_g2`: header checks as parse_ptau_file, both records on the twist).  Host only."""
    lib = _lib.load()
    h, beta_h = np.zeros(16, dtype=np.uint64), np.zeros(16, dtype=np.uint64)
    _lib.check(lib.b200_srs_parse_ptau_g2(data, len(data), _ptr(h), _ptr(beta_h)))
    return h, beta_h


def parse_ptau_file(ctx: Context, data: bytes, window_bits: int = 0,
                    check_on_curve: bool = True, count: int | None = None) -> UnivariateUniversalParams:
    """srs.rs:63-71: header/section checks, MAX_SRS_DEGREE+1 G1 powers, on-curve assertion
    (srs.rs:178-179, run on the device).  `count` overrides the number of powers kept (the
    reference always keeps MAX_SRS_DEGREE + 1; smaller values serve truncated test files).  `h` / `beta_h` are read
    from section 3 when the file holds it (read_ptau_g2), else left None; a G2 record there off the twist raises."""
    lib = _lib.load()
    buf = (C.c_char * len(data)).from_buffer_copy(data)
    rec = C.c_void_p()
    n = C.c_size_t()
    _lib.check(lib.b200_srs_parse_ptau(C.cast(buf, C.c_void_p), len(data), C.byref(rec), C.byref(n)))
    need = MAX_SRS_DEGREE + 1 if count is None else count
    if n.value < need:
        raise _lib.B200Error(_lib.B200_ERR_FORMAT, f"ptau: only {n.value} G1 records available, need {need}")
    try:
        g2 = read_ptau_g2(data)
    except _lib.B200Error as e:  # no section 3 (the truncated files accepted above): no G2 pair; a bad record raises
        if e.code != _lib.B200_ERR_FORMAT:
            raise
        g2 = (None, None)
    off = rec.value - C.addressof(buf)
    host = np.frombuffer(data, dtype=np.uint64, count=need * 8, offset=off).reshape(need, 8).copy()
    bases = ctx.load_bases(host, window_bits=window_bits, check_on_curve=check_on_curve)
    return UnivariateUniversalParams(powers_of_g=bases, powers_of_g_host=host, h=g2[0], beta_h=g2[1])


def g2_in_subgroup(rec) -> bool:
    """[r]Q == O for a 128-byte G2 record (`b200_g2_in_subgroup`; the identity is not in the subgroup).  Host only."""
    out = C.c_int(0)
    _lib.check(_lib.load().b200_g2_in_subgroup(_ptr(_u64(rec, 16)), C.byref(out)))
    return bool(out.value)


SRS_REPORT_MAX_BAD = 8  # failing pair indices b200_srs_report lists


@dataclass
class SrsReport:
    """`b200_srs_report`: the SRS is valid exactly when `valid` (consistent powers, P_0 = G, h and beta_h of order r).
    `bad` lists the first failing pairs (P_i, P_{i+1}) by i, ascending, of `n_bad` in all (located only on request)."""
    consistent: bool
    g1_generator: bool
    g2_subgroup: bool
    n_bad: int
    bad: list

    @property
    def valid(self) -> bool:
        return self.consistent and self.g1_generator and self.g2_subgroup


def check_srs(ctx: Context, bases: Bases, h, beta_h, n: int | None = None, seed: bytes | None = None,
              locate: bool = True) -> SrsReport:
    """Checks that the first n (default: all) loaded powers are tau^i G for the tau of beta_h = tau h, with one batch-2
    MSM on the device and one pairing (`b200_srs_check`).  The weights are the powers of a rho drawn from `seed`
    (32 bytes; None draws `secrets.token_bytes(32)`), which must be unknown to whoever made the file.  With `locate`,
    a failed check is followed by every consecutive pair checked on its own on the device, which fills `n_bad` / `bad`."""
    import secrets
    n = len(bases) if n is None else n
    seed = secrets.token_bytes(32) if seed is None else bytes(seed)
    if len(seed) != 32:
        raise ValueError("seed: 32 bytes")
    rep = _lib.STRUCTS["b200_srs_report"]()
    _lib.check(ctx._lib.b200_srs_check(ctx._h, bases._h, n, _ptr(_u64(h, 16)), _ptr(_u64(beta_h, 16)), seed, int(locate),
                                       C.byref(rep)))
    return SrsReport(consistent=bool(rep.consistent), g1_generator=bool(rep.g1_generator), g2_subgroup=bool(rep.g2_subgroup),
                     n_bad=int(rep.n_bad), bad=[int(rep.bad[i]) for i in range(min(int(rep.n_bad), SRS_REPORT_MAX_BAD))])


class VariableBaseMSM:
    """ark-ec 0.4.2 `VariableBaseMSM`."""

    @staticmethod
    def msm_bigint(ctx: Context, bases: Bases, bigints: np.ndarray):
        """sum_i bigints[i] * bases[i]; bigints canonical (`BigInt<4>`).  Returns the affine
        result (x||y Montgomery, identity flag) — what `.into_affine()` yields."""
        return ctx.msm(bases, bigints, montgomery=False)


class UnivariateKzgPCS:
    """jf-primitives `UnivariateKzgPCS`."""

    @staticmethod
    def commit(ctx: Context, prover_param: Bases, poly_coeffs: np.ndarray):
        """Commitment to a dense polynomial given by Montgomery `Fr` coefficients: the
        Montgomery->canonical conversion jf-primitives does on the CPU
        (`convert_to_bigints`) is fused into the device digit extraction."""
        return ctx.msm(prover_param, poly_coeffs, montgomery=True)


class Radix2EvaluationDomain:
    """ark-poly 0.4.2 `Radix2EvaluationDomain<Fr>`: natural order in and out."""

    def __init__(self, ctx: Context, num_coeffs: int):
        size = 1
        while size < num_coeffs:
            size <<= 1
        self.ctx = ctx
        self.size = size
        self.log_size_of_group = size.bit_length() - 1
        self.group_gen = ctx.domain_generator(self.log_size_of_group)

    def _pad(self, x: np.ndarray) -> np.ndarray:
        x = np.ascontiguousarray(x, dtype=np.uint64).reshape(-1, 4)
        if x.shape[0] > self.size:
            raise ValueError("more coefficients than the domain size")
        if x.shape[0] < self.size:  # ark-poly resizes with zeros
            x = np.concatenate([x, np.zeros((self.size - x.shape[0], 4), dtype=np.uint64)])
        return x

    def fft(self, coeffs: np.ndarray) -> np.ndarray:
        return self.ctx.ntt(self._pad(coeffs), inverse=False, coset=False)

    def ifft(self, evals: np.ndarray) -> np.ndarray:
        return self.ctx.ntt(self._pad(evals), inverse=True, coset=False)

    def coset_fft(self, coeffs: np.ndarray) -> np.ndarray:
        return self.ctx.ntt(self._pad(coeffs), inverse=False, coset=True)

    def coset_ifft(self, evals: np.ndarray) -> np.ndarray:
        return self.ctx.ntt(self._pad(evals), inverse=True, coset=True)


# ---------------------------------------------------------------------------------------------
# TurboPlonk prover (boundary B2)
# ---------------------------------------------------------------------------------------------
class B200Proof(_lib.STRUCTS["b200_proof"]):
    """b200_proof: field order of the reference's `PlonkProof` (plonk_proof_def.rs:197-222)."""

    def to_array(self) -> np.ndarray:
        return np.frombuffer(bytes(self), dtype=np.uint64).copy()


@dataclass
class LinkingHint:
    """mpc-plonk `LinkingHint` (plonk_proof_def.rs:143-150)."""
    linking_wire_poly: np.ndarray
    linking_wire_comm: np.ndarray


class ProvingKey:
    """Device-resident `ProvingKey` + the `VerifyingKey` commitments (b200_pk)."""

    def __init__(self, ctx: Context, handle, log_n: int, num_inputs: int, k: np.ndarray):
        self._ctx, self._h = ctx, handle
        self.log_n, self.num_inputs, self.k = log_n, num_inputs, k
        self.selector_comms = np.zeros((13, 8), dtype=np.uint64)
        self.sigma_comms = np.zeros((5, 8), dtype=np.uint64)
        _lib.check(ctx._lib.b200_pk_verifying_key(handle, _ptr(self.selector_comms), _ptr(self.sigma_comms)))

    @property
    def domain_size(self) -> int:
        return 1 << self.log_n

    @property
    def num_vars(self) -> int:
        """Length of the witness vector a proof of this key takes; 0 for a key without wiring (`preprocess`)."""
        return int(self._ctx._lib.b200_pk_num_vars(self._h))

    @property
    def compact(self) -> bool:
        """True for a key made with compact=True (b200compact.h): no coset tables, round 3 one coset at a time."""
        return bool(self._ctx._lib.b200_pk_is_compact(self._h))

    def free(self):
        if self._h:
            self._ctx._lib.b200_pk_free(self._ctx._h, self._h)
        self._h = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


@dataclass
class VerifyingKey:
    """mpc-plonk `VerifyingKey<Bn254>` flattened: domain size, public-input count, coset representatives, the 13
    selector and 5 sigma commitments, and the two G2 elements of the `open_key` (`h`, `beta_h`: 128-byte ptau
    records x0 || x1 || y0 || y1, srs.rs:185-199).  Plain host data: verification needs no device."""
    log_n: int
    num_inputs: int
    k: np.ndarray
    selector_comms: np.ndarray
    sigma_comms: np.ndarray
    g2_h: np.ndarray
    g2_tau_h: np.ndarray

    @staticmethod
    def from_proving_key(pk: "ProvingKey", g2_h: np.ndarray, g2_tau_h: np.ndarray) -> "VerifyingKey":
        return VerifyingKey(pk.log_n, pk.num_inputs, pk.k, pk.selector_comms, pk.sigma_comms, g2_h, g2_tau_h)


B200VerifyingKey = _lib.STRUCTS["b200_verifying_key"]  # the flat verifying key of b200_plonk_verify
B200BatchProof = _lib.STRUCTS["b200_batch_proof"]      # one proof of a batch (index of its key, public inputs, proof)
B200BatchLink = _lib.STRUCTS["b200_batch_link"]        # one link proof of a batch


def _u64(a, shape=None) -> np.ndarray:
    a = np.ascontiguousarray(a, dtype=np.uint64)
    return a.reshape(shape) if shape is not None else a


PAIRING_MAX_PAIRS = 8  # pairs per check of b200_pairing_check_many


def pairing_check(g1_points, g2_points) -> bool:
    """prod e(P_i, Q_i) == 1 (`b200_pairing_check`; host only).  P_i: 8 x uint64, Q_i: 16 x uint64."""
    lib = _lib.load()
    p = _u64(np.stack([_u64(x) for x in g1_points]), (-1, 8))
    q = _u64(np.stack([_u64(x) for x in g2_points]), (-1, 16))
    if p.shape[0] != q.shape[0]:
        raise ValueError("one G2 point per G1 point")
    one = C.c_int(0)
    _lib.check(lib.b200_pairing_check(_ptr(p), _ptr(q), p.shape[0], C.byref(one)))
    return bool(one.value)


def pairing_check_many(ctx: Context, g2_points, g1_points) -> np.ndarray:
    """n independent pairing checks against the same m G2 points on `ctx`'s device (`b200_pairing_check_many`):
    out[c] = prod_j e(g1_points[c, j], g2_points[j]) == 1.  g2_points: (m, 16) uint64, g1_points: (n, m, 8) uint64,
    m <= PAIRING_MAX_PAIRS.  Each answer equals `pairing_check` over the check's m pairs."""
    q = _u64(g2_points)
    if q.ndim != 2 or q.shape[1] != 16:
        raise ValueError("g2_points: (m, 16) uint64")
    m = q.shape[0]
    p = _u64(g1_points)
    if p.ndim != 3 or p.shape[1:] != (m, 8):
        raise ValueError("g1_points: (n, m, 8) uint64 with m = len(g2_points)")
    if m > PAIRING_MAX_PAIRS:
        raise ValueError("at most %d pairs per check" % PAIRING_MAX_PAIRS)
    n = p.shape[0]
    out = np.zeros(max(1, n), dtype=np.uint8)
    _lib.check(ctx._lib.b200_pairing_check_many(ctx._h, _ptr(q) if m else None, m, _ptr(p) if p.size else None, n,
                                                 out.ctypes.data_as(C.c_void_p)))
    return out[:n].astype(bool)


def verify_link_proof(comm_a: np.ndarray, comm_b: np.ndarray, proof: "B200LinkProof", layout: "GroupLayout",
                      g2_h: np.ndarray, g2_tau_h: np.ndarray) -> bool:
    """`PlonkKzgSnark::verify_link_proof::<SolidityTranscript>` (proof_linking/intent_only.rs:77-84)."""
    ok = C.c_int(0)
    _lib.check(_lib.load().b200_plonk_verify_link(_ptr(_u64(comm_a)), _ptr(_u64(comm_b)), layout.alignment, layout.offset,
                                                  layout.size, C.byref(proof), _ptr(_u64(g2_h)), _ptr(_u64(g2_tau_h)),
                                                  C.byref(ok)))
    return bool(ok.value)


class _VerifyBatch:
    """The Python argument checks and the C structs of `batch_verify` and `verify_each`: the distinct verifying keys, the
    proofs whose public-input count matches their key (the others are False verdicts without a device call), the
    links and the one G2 pair.  `args` are the C call's arguments from ctx on, up to the outputs; `where`, the entry point,
    starts the message of a refused link."""

    def __init__(self, vks, pub_inputs, proofs, links, g2, where: str = "verify"):
        vks, pub_inputs, proofs, links = list(vks), list(pub_inputs), list(proofs), list(links)
        if not (len(vks) == len(pub_inputs) == len(proofs)):
            raise ValueError("one verifying key and one public-input vector per proof")
        g2_pairs = {(_u64(vk.g2_h).tobytes(), _u64(vk.g2_tau_h).tobytes()) for vk in vks}
        if g2 is not None:
            g2_pairs.add((_u64(g2[0]).tobytes(), _u64(g2[1]).tobytes()))
        if len(g2_pairs) > 1:
            raise ValueError("the verifying keys of one batch must share the G2 pair (h, beta_h)")
        self.n_proofs = len(proofs)
        self.n_items = len(proofs) + len(links)
        if not g2_pairs:
            if self.n_items:
                raise ValueError("links without proofs need g2=(g2_h, g2_tau_h)")
            return
        g2_h, g2_tau_h = (np.frombuffer(b, dtype=np.uint64).copy() for b in next(iter(g2_pairs)))
        self.keep = [g2_h, g2_tau_h]  # the arrays the C structs point into stay alive as long as this object
        # distinct verifying keys
        vk_index, c_vks = {}, []
        for vk in vks:
            arrs = (_u64(vk.k, (5, 4)), _u64(vk.selector_comms, (13, 8)), _u64(vk.sigma_comms, (5, 8)))
            key = (vk.log_n, vk.num_inputs) + tuple(a.tobytes() for a in arrs)
            if key not in vk_index:
                vk_index[key] = len(c_vks)
                self.keep.append(arrs)
                c_vks.append(B200VerifyingKey(vk.log_n, vk.num_inputs, *(_ptr(a) for a in arrs)))
        c_proofs, self.proof_pos = [], []
        for i, (vk, pi, proof) in enumerate(zip(vks, pub_inputs, proofs)):
            p = _u64(pi, (-1, 4))
            if p.shape[0] != vk.num_inputs:
                continue  # not accepted (the reference's verifier errors on a wrong public-input count)
            self.keep.append(p)
            key = (vk.log_n, vk.num_inputs) + tuple(
                a.tobytes() for a in (_u64(vk.k, (5, 4)), _u64(vk.selector_comms, (13, 8)), _u64(vk.sigma_comms, (5, 8))))
            c_proofs.append(B200BatchProof(vk_index[key], _ptr(p) if p.size else None, C.cast(C.pointer(proof), C.c_void_p)))
            self.proof_pos.append(i)
        c_links = []
        for i, (comm_a, comm_b, lproof, layout) in enumerate(links):
            _check_group_size(layout, f"{where}: link {i}")
            a, b = _u64(comm_a), _u64(comm_b)
            self.keep.append((a, b))
            c_links.append(B200BatchLink(_ptr(a), _ptr(b), layout.alignment, layout.offset, layout.size,
                                         C.cast(C.pointer(lproof), C.c_void_p)))
        self.c_proofs, self.c_links = c_proofs, c_links
        self.n_c = len(c_proofs) + len(c_links)
        arrays = ((B200VerifyingKey * max(1, len(c_vks)))(*c_vks), (B200BatchProof * max(1, len(c_proofs)))(*c_proofs),
                  (B200BatchLink * max(1, len(c_links)))(*c_links))
        self.keep.append(arrays)
        self.args = (arrays[0], len(c_vks), arrays[1], len(c_proofs), arrays[2], len(c_links), _ptr(g2_h), _ptr(g2_tau_h))

    def verdicts(self, c_verdicts) -> list:
        """The C call's verdicts at the caller's item positions; a proof left out is False."""
        out = [False] * self.n_items
        for j, i in enumerate(self.proof_pos):
            out[i] = bool(c_verdicts[j])
        for j in range(len(self.c_links)):
            out[self.n_proofs + j] = bool(c_verdicts[len(self.c_proofs) + j])
        return out


class PlonkKzgSnark:
    """mpc-plonk `PlonkKzgSnark<Bn254>` as called at traits.rs:850, traits.rs:996 and traits.rs:1012."""

    @staticmethod
    def verify(vk: VerifyingKey, pub_inputs: np.ndarray, proof: "B200Proof") -> bool:
        """`PlonkKzgSnark::verify::<SolidityTranscript>(&vk, &public_inputs, &proof, None)` (traits.rs:1012-1018).
        Host only."""
        pi = _u64(pub_inputs, (-1, 4))
        if pi.shape[0] != vk.num_inputs:
            return False  # the reference's verifier errors on a wrong public-input count: not accepted
        ok = C.c_int(0)
        _lib.check(_lib.load().b200_plonk_verify(vk.log_n, vk.num_inputs, _ptr(_u64(vk.k, (5, 4))),
                                                 _ptr(_u64(vk.selector_comms, (13, 8))), _ptr(_u64(vk.sigma_comms, (5, 8))),
                                                 _ptr(pi) if pi.size else None, C.byref(proof), _ptr(_u64(vk.g2_h)),
                                                 _ptr(_u64(vk.g2_tau_h)), C.byref(ok)))
        return bool(ok.value)

    @staticmethod
    def batch_verify(ctx: Context, vks, pub_inputs, proofs, links=(), g2=None):
        """Verifies many proofs and link proofs with ONE pairing on `ctx`'s device (`b200_plonk_batch_verify`).

        vks[i], pub_inputs[i], proofs[i]: the arguments of `verify` for proof i; links: (comm_a, comm_b, B200LinkProof,
        GroupLayout) tuples, the arguments of `verify_link_proof`.  Every key must carry the same G2 pair (else
        ValueError); `g2 = (g2_h, g2_tau_h)` supplies it when there are only links.  Returns (all_ok, verdicts) with
        verdicts[i] the single verifier's answer for item i, proofs first, then links.  A wrong public-input count is
        a False verdict, as in `verify`."""
        b = _VerifyBatch(vks, pub_inputs, proofs, links, g2, "batch_verify")
        if b.n_items == 0:
            return True, []
        verdicts = (C.c_uint8 * max(1, b.n_c))()
        ok = C.c_int(0)
        _lib.check(ctx._lib.b200_plonk_batch_verify(ctx._h, *b.args, C.byref(ok), verdicts))
        return bool(ok.value) and len(b.c_proofs) == b.n_proofs, b.verdicts(verdicts)

    @staticmethod
    def verify_each(ctx: Context, vks, pub_inputs, proofs, links=(), g2=None) -> list:
        """The verdicts of `batch_verify`, each item checked on its own with its own pairing on `ctx`'s device
        (`b200_plonk_verify_each`): no bisection, so the cost does not depend on how many items fail.  Same arguments
        and argument errors as `batch_verify`; returns the list of verdicts, proofs first, then links."""
        b = _VerifyBatch(vks, pub_inputs, proofs, links, g2, "verify_each")
        if b.n_items == 0:
            return []
        verdicts = (C.c_uint8 * max(1, b.n_c))()
        _lib.check(ctx._lib.b200_plonk_verify_each(ctx._h, *b.args, verdicts))
        return b.verdicts(verdicts)

    @staticmethod
    def preprocess(ctx: Context, srs: Bases, log_n: int, num_inputs: int, selectors: np.ndarray,
                   perm: np.ndarray, k: np.ndarray, compact: bool = False) -> ProvingKey:
        """compact=True: a compact key (b200_plonk_preprocess_compact), the same verifying key and proofs from a fraction
        of the device memory (`footprint`), at the cost of round-3 time."""
        sel = np.ascontiguousarray(selectors, dtype=np.uint64).reshape(13, 1 << log_n, 4)
        pm = np.ascontiguousarray(perm, dtype=np.uint64).reshape(5 << log_n)
        kk = np.ascontiguousarray(k, dtype=np.uint64).reshape(5, 4)
        h = C.c_void_p()
        fn = ctx._lib.b200_plonk_preprocess_compact if compact else ctx._lib.b200_plonk_preprocess
        _lib.check(fn(ctx._h, srs._h, log_n, num_inputs, _ptr(sel), _ptr(pm), _ptr(kk), C.byref(h)))
        return ProvingKey(ctx, h, log_n, num_inputs, kk)

    @staticmethod
    def preprocess_wiring(ctx: Context, srs: Bases, log_n: int, num_inputs: int, selectors: np.ndarray,
                          wire_vars: np.ndarray, num_vars: int, k: np.ndarray, compact: bool = False) -> ProvingKey:
        """`preprocess` from the circuit's wiring (b200_plonk_preprocess_wiring): wire_vars[i, j] = the variable on wire i of
        row j (5 x n, < num_vars).  The copy permutation is derived on the device and the key keeps the wiring, so its
        proofs are made from witness vectors (`prove_witness`).  compact=True as for `preprocess`."""
        sel = np.ascontiguousarray(selectors, dtype=np.uint64).reshape(13, 1 << log_n, 4)
        wv = np.ascontiguousarray(wire_vars, dtype=np.uint32).reshape(5 << log_n)
        kk = np.ascontiguousarray(k, dtype=np.uint64).reshape(5, 4)
        h = C.c_void_p()
        fn = ctx._lib.b200_plonk_preprocess_wiring_compact if compact else ctx._lib.b200_plonk_preprocess_wiring
        _lib.check(fn(ctx._h, srs._h, log_n, num_inputs, _ptr(sel), wv.ctypes.data_as(C.c_void_p), num_vars, _ptr(kk), C.byref(h)))
        return ProvingKey(ctx, h, log_n, num_inputs, kk)

    FOOTPRINT_PARTS = ("key", "ntt_scratch", "domain", "srs", "msm_scratch", "runtime", "workspace", "ntt_scratch2",
                       "batch_workspace", "batch_ntt_scratch", "batch_ntt_scratch2", "batch_msm_scratch")

    @staticmethod
    def footprint(log_n: int, k: int = 1, compact: bool = False) -> dict:
        """b200_plonk_footprint: the device bytes of one context with one key of domain 2^log_n and a call of k proofs,
        {part: bytes} in the header's order.  Needs no device."""
        out = (C.c_uint64 * _lib.FOOTPRINT_PARTS)()
        _lib.check(_lib.load().b200_plonk_footprint(log_n, k, int(compact), out))
        return dict(zip(PlonkKzgSnark.FOOTPRINT_PARTS, (int(v) for v in out)))

    @staticmethod
    def prove_witness(ctx: Context, pk: ProvingKey, witness, blinders: np.ndarray, want_challenges: bool = False):
        """`prove_with_link_hint` from the witness vector (b200_plonk_prove_witness) of a key made by `preprocess_wiring`:
        witness is the num_vars x 4 array, or the address of one in device or pinned host memory (int).  Returns
        (proof, LinkingHint, pub_inputs[, challenges]); proof, hint and challenges equal `prove_with_link_hint` on the
        expanded wire table."""
        p = _witness_proof(pk, witness, blinders, "prove_witness", link=True, challenges=True)
        _lib.check(ctx._lib.b200_plonk_prove_witness(ctx._h, pk._h, p.src, _ptr(p.bl), C.byref(p.proof), _ptr(p.link),
                                                     _ptr(p.challenges) if want_challenges else None, _opt(p.pub)))
        return (p.proof, p.hint(), p.pub, p.challenges) if want_challenges else (p.proof, p.hint(), p.pub)

    @staticmethod
    def prove_witness_batch(ctx: Context, pk: ProvingKey, witness_list, blinders_list, link_hints: bool = False,
                            want_challenges: bool = False):
        """`prove_batch` with the items given as witness vectors (b200_plonk_prove_witness_batch).  Returns
        (proofs, hints, statuses, pub_inputs[, challenges]), item i as `prove_witness` of the same arguments."""
        items, ps = _witness_items(pk, witness_list, blinders_list, link_hints, want_challenges, "prove_witness_batch")
        statuses = (C.c_int * max(1, len(ps)))()
        rc = ctx._lib.b200_plonk_prove_witness_batch(ctx._h, pk._h, items, len(ps), statuses)
        if rc not in (_lib.B200_OK, _lib.B200_ERR_UNSATISFIED):
            _lib.check(rc)
        res = _batch_results(ps, statuses, link_hints, want_challenges)
        return res[:3] + ([p.pub for p in ps],) + res[3:]

    @staticmethod
    def prove_with_link_hint(ctx: Context, pk: ProvingKey, wires: np.ndarray, pub_inputs: np.ndarray,
                             blinders: np.ndarray, want_challenges: bool = False):
        """Returns (proof, LinkingHint[, challenges]).  `blinders` are the 17 field elements the
        reference draws from `thread_rng()` (traits.rs:994), in draw order."""
        p = _table_proof(pk, wires, pub_inputs, blinders, "prove_with_link_hint", link=True, challenges=True)
        _lib.check(ctx._lib.b200_plonk_prove(ctx._h, pk._h, p.src, _opt(p.pub), _ptr(p.bl), C.byref(p.proof), _ptr(p.link),
                                             _ptr(p.challenges) if want_challenges else None))
        return (p.proof, p.hint(), p.challenges) if want_challenges else (p.proof, p.hint())

    @staticmethod
    def prove_batch(ctx: Context, pk: ProvingKey, wires_list, pub_inputs_list, blinders_list, link_hints: bool = False,
                    want_challenges: bool = False):
        """Proves k witnesses of one key in ONE call (`b200_plonk_prove_batch`): every launch covers all k proofs and every
        commitment round is one batched MSM.  wires_list[i]: a 5 x n wire table (array) or the address of one in device or
        pinned host memory (int); pub_inputs_list[i], blinders_list[i]: as for `prove_with_link_hint`.  Returns
        (proofs, hints, statuses[, challenges]): item i's proof, hint and challenges equal `prove_with_link_hint` of the same
        arguments; statuses[i] is 0, or -7 (B200_ERR_UNSATISFIED) for a witness that does not satisfy the circuit, whose
        proof is zeroed and whose hint is None (hints is None without link_hints).  Argument errors raise ValueError before
        any device work; other failures raise B200Error."""
        items, ps = _prove_items(pk, wires_list, pub_inputs_list, blinders_list, link_hints, want_challenges, "prove_batch")
        statuses = (C.c_int * max(1, len(ps)))()
        rc = ctx._lib.b200_plonk_prove_batch(ctx._h, pk._h, items, len(ps), statuses)
        if rc not in (_lib.B200_OK, _lib.B200_ERR_UNSATISFIED):
            _lib.check(rc)
        return _batch_results(ps, statuses, link_hints, want_challenges)

    @staticmethod
    def prove_settlement(ctx: Context, srs: Bases, pk: ProvingKey, wires, pub_inputs, blinders, links):
        """A settlement in ONE call (`b200_plonk_prove_settlement`): proves the statement, then links every stored hint to
        the statement's own hint as one link batch.  wires: the 5 x n table (array) or its address in device or pinned
        host memory (int); links = [(LinkingHint, GroupLayout)], each hint's linking_wire_poly an array or (address,
        length) of one in device or pinned host memory.  Returns (proof, link_proofs, statuses): the proof equals
        `prove_with_link_hint`'s, link i equals `link_proofs(hint_i, settlement hint, layout_i)`; statuses[0] is the
        proof's, statuses[1 + i] link i's (0, or -7 = B200_ERR_UNSATISFIED: an unsatisfied witness zeroes everything, a
        stale hint zeroes its own link proof).  Argument errors raise ProverError before any library call."""
        (e, arr, n_links, st), finish, _ = _settlement_job(pk._h, pk, len(srs), links, _table_proof, wires, pub_inputs,
                                                           blinders, where="prove_settlement")
        e = e.contents
        rc = ctx._lib.b200_plonk_prove_settlement(ctx._h, srs._h, pk._h, e.wires, e.pub_inputs, e.blinders, e.proof,
                                                  e.link_poly, arr, n_links, st)
        return finish(rc)

    @staticmethod
    def prove_settlement_witness(ctx: Context, srs: Bases, pk: ProvingKey, witness, blinders, links):
        """`prove_settlement` from the settlement's witness vector (`b200_plonk_prove_settlement_witness`) of a key made by
        `preprocess_wiring`: witness as `prove_witness` takes it.  Returns (proof, link_proofs, statuses, pub_inputs)."""
        (e, arr, n_links, st), finish, _ = _settlement_job(pk._h, pk, len(srs), links, _witness_proof, witness, blinders,
                                                           where="prove_settlement_witness")
        e = e.contents
        rc = ctx._lib.b200_plonk_prove_settlement_witness(ctx._h, srs._h, pk._h, e.witness, e.blinders, e.proof,
                                                          e.link_poly, e.pub_inputs_out, arr, n_links, st)
        return finish(rc)


B200ProveItem = _lib.STRUCTS["b200_prove_item"]  # one witness of a batch
B200WitnessItem = _lib.STRUCTS["b200_witness_item"]  # one witness vector of a batch


# ---- proof and link inputs -----------------------------------------------------------------------------------------
# Every entry point that takes a proof or a link builds it with `_table_proof`, `_witness_proof` or `_link_item`.  They
# check the input against the key's shape (`domain_size`, `num_inputs`, `num_vars` of a ProvingKey or a box key) and raise
# ValueError before any library call, since the library reads fixed-size arrays through the pointers it is given.  A
# message names the entry point, then the item, proof or link, then the field and the numbers.  Entry points that
# refuse with ProverError convert in `_prover_errors`.

def _opt(a):
    """Pointer to an array, or NULL for no array or an empty one."""
    return _ptr(a) if a is not None and a.size else None


def _prover_errors(build):
    """`build` with its argument errors (ValueError) raised as ProverError(B200_ERR_INVALID)."""
    @functools.wraps(build)
    def checked(*args, **kwargs):
        try:
            return build(*args, **kwargs)
        except ValueError as e:
            raise ProverError(_lib.B200_ERR_INVALID, str(e)) from None
    return checked


class _Proof(NamedTuple):
    """One proof's checked inputs and the buffers the prover writes: `proof`, and the (n + 2, 4) `link` polynomial and
    (6, 4) `challenges` when asked for (else None).  `held` is the wire table or witness array (None for an address),
    `src` the pointer to it.  `pub` is a wire-table proof's public inputs, or the array a witness proof's public inputs
    are written to."""
    held: object
    pub: np.ndarray
    bl: np.ndarray
    proof: B200Proof
    link: object
    challenges: object
    src: object
    witness: bool

    def _proof_ptr(self):
        return C.cast(C.pointer(self.proof), C.c_void_p)

    def item(self):
        """The proof as an item of a context batch: b200_witness_item or b200_prove_item."""
        if self.witness:
            return B200WitnessItem(self.src, _ptr(self.bl), self._proof_ptr(), _opt(self.link), _opt(self.challenges),
                                   _opt(self.pub))
        return B200ProveItem(self.src, _opt(self.pub), _ptr(self.bl), self._proof_ptr(), _opt(self.link),
                             _opt(self.challenges))

    def entry(self, pk):
        """The proof as an entry of a pool job, key handle `pk`: b200_bundle_witness or b200_bundle_proof."""
        if self.witness:
            return BundleWitness(pk, self.src, _ptr(self.bl), self._proof_ptr(), _opt(self.link), _opt(self.pub))
        return BundleProof(pk, self.src, _opt(self.pub), self.pub.shape[0], _ptr(self.bl), self._proof_ptr(),
                           _opt(self.link))

    def hint(self):
        return LinkingHint(linking_wire_poly=self.link, linking_wire_comm=np.array(self.proof.wires_poly_comms[0],
                                                                                   dtype=np.uint64))


def _proof(shape, witness: bool, src, held, pub, blinders, link: bool, challenges: bool, where: str) -> _Proof:
    """A `_Proof` with its blinders checked and its output buffers made."""
    bl = np.ascontiguousarray(blinders, dtype=np.uint64)
    if bl.size != 17 * 4:
        raise ValueError(f"{where} has {bl.size // 4} blinders, the prover draws 17: blinders must be 17 Fr elements")
    return _Proof(held, pub, bl, B200Proof(),
                  np.zeros((shape.domain_size + 2, 4), dtype=np.uint64) if link else None,
                  np.zeros((6, 4), dtype=np.uint64) if challenges else None, src, witness)


def _table_proof(shape, wires, pub_inputs, blinders, where: str, link: bool = False, challenges: bool = False) -> _Proof:
    """A proof of a 5 x n wire table, given as an array or as the address of one in device or pinned host memory."""
    if isinstance(wires, (int, np.integer)):
        w, src = None, C.c_void_p(int(wires))
    else:
        w = np.ascontiguousarray(wires, dtype=np.uint64)
        if w.size != 5 * shape.domain_size * 4:
            raise ValueError(f"{where}: the wire table has {w.size // 4} elements, the key needs 5 x {shape.domain_size}")
        src = _ptr(w)
    pi = np.ascontiguousarray(pub_inputs, dtype=np.uint64)
    if pi.size != 4 * shape.num_inputs:
        raise ValueError(f"{where} has {pi.size // 4} public inputs for a key with {shape.num_inputs}: public inputs / "
                         "blinders do not match the key")
    return _proof(shape, False, src, w, pi.reshape(-1, 4), blinders, link, challenges, where)


def _witness_proof(shape, witness, blinders, where: str, link: bool = False, challenges: bool = False) -> _Proof:
    """A proof of a witness vector of a key made by `preprocess_wiring`, given as an array of the key's num_vars elements or
    as the address of one in device or pinned host memory.  A key without wiring is ProverError, as the library says."""
    if shape.num_vars == 0:
        raise ProverError(_lib.B200_ERR_INVALID, f"{where} holds no wiring: its key was made by preprocess")
    if isinstance(witness, (int, np.integer)):
        wit, src = None, C.c_void_p(int(witness))
    else:
        wit = np.ascontiguousarray(witness, dtype=np.uint64)
        if wit.size != 4 * shape.num_vars:
            raise ValueError(f"{where}: the witness has {wit.size // 4} elements, the key takes {shape.num_vars}")
        src = _ptr(wit)
    pub = np.zeros((shape.num_inputs, 4), dtype=np.uint64)
    return _proof(shape, True, src, wit, pub, blinders, link, challenges, where)


def _witness_items(pk, witness_list, blinders_list, link_hints: bool, want_challenges: bool, where: str):
    """A witness batch: (its b200_witness_item array, the `_Proof` of each item)."""
    witness_list, blinders_list = list(witness_list), list(blinders_list)
    if len(witness_list) != len(blinders_list):
        raise ValueError(f"{where}: {len(witness_list)} witness vectors and {len(blinders_list)} blinder vectors")
    ps = [_witness_proof(pk, w, b, f"{where}: item {i}", link_hints, want_challenges)
          for i, (w, b) in enumerate(zip(witness_list, blinders_list))]
    return (B200WitnessItem * max(1, len(ps)))(*(p.item() for p in ps)), ps


def _prove_items(pk, wires_list, pub_inputs_list, blinders_list, link_hints: bool, want_challenges: bool,
                 where: str = "prove_batch"):
    """A batch of wire tables: (its b200_prove_item array, the `_Proof` of each item)."""
    wires_list, pub_inputs_list, blinders_list = list(wires_list), list(pub_inputs_list), list(blinders_list)
    k = len(wires_list)
    if len(pub_inputs_list) != k or len(blinders_list) != k:
        raise ValueError(f"{where}: {k} wire tables, {len(pub_inputs_list)} public-input vectors and "
                         f"{len(blinders_list)} blinder vectors: one of each per witness")
    ps = [_table_proof(pk, w, pi, b, f"{where}: item {i}", link_hints, want_challenges)
          for i, (w, pi, b) in enumerate(zip(wires_list, pub_inputs_list, blinders_list))]
    return (B200ProveItem * max(1, k))(*(p.item() for p in ps)), ps


def _batch_results(ps, statuses, link_hints: bool, want_challenges: bool):
    st = [int(statuses[i]) for i in range(len(ps))]
    hints = [p.hint() if s == _lib.B200_OK else None for p, s in zip(ps, st)] if link_hints else None
    if want_challenges:
        return [p.proof for p in ps], hints, st, [p.challenges for p in ps]
    return [p.proof for p in ps], hints, st


def _link_hint(hint, where: str, name: str):
    """(pointer, length, array or None, commitment) of `where`'s hint `name`: its polynomial is an array of (len, 4) limbs,
    or (address, len) of one in device or pinned host memory; its commitment is 8 limbs (x || y)."""
    poly = hint.linking_wire_poly
    if isinstance(poly, tuple):
        addr, n = poly
        p, n, a = C.c_void_p(int(addr)), int(n), None
    else:
        a = np.ascontiguousarray(poly, dtype=np.uint64)
        if a.size % 4:
            raise ValueError(f"{where}'s {name} is not a vector of field elements (4 limbs each)")
        a = a.reshape(-1, 4)
        p, n = _ptr(a), a.shape[0]
    c = np.ascontiguousarray(hint.linking_wire_comm, dtype=np.uint64).reshape(-1)
    if c.size != 8:
        raise ValueError(f"{where}'s {name} commitment must be 8 limbs (x || y), not {c.size}")
    return p, n, a, c


def _check_group_size(lay: "GroupLayout", where: str):
    """`where`'s link group holds distinct roots: at most the 2^alignment of its subgroup (an alignment outside [0, 28] is
    left to the caller's other checks)."""
    if 0 <= lay.alignment <= 28 and lay.size > 1 << lay.alignment:
        raise ValueError(f"{where}'s group of {lay.size} roots does not fit the 2^{lay.alignment} roots of unity of its "
                         "alignment (size <= 2^alignment)")


def _check_layout(lay: "GroupLayout", length: int, srs_len, where: str):
    """`where`'s link group on polynomials of `length` coefficients, against an SRS of `srs_len` powers (None: not known
    here)."""
    if not 0 < lay.size < length:
        raise ValueError(f"{where}'s group of {lay.size} roots does not fit polynomials of {length} coefficients "
                         "(0 < size < length)")
    if not 0 <= lay.alignment <= 28 or lay.offset < 0:
        raise ValueError(f"{where} has alignment {lay.alignment} and offset {lay.offset} (0 <= alignment <= 28, offset >= 0)")
    _check_group_size(lay, where)
    if srs_len is not None and length > srs_len:
        raise ValueError(f"{where} has {length} coefficients, the SRS {srs_len} powers")


def keccak256(data: bytes) -> bytes:
    out = (C.c_uint8 * 32)()
    _lib.load().b200_keccak256(data, len(data), out)
    return bytes(out)


def plonk_last_timings(ctx: Context) -> dict:
    arr = (C.c_float * 8)()
    _lib.check(ctx._lib.b200_plonk_last_timings(ctx._h, C.byref(arr)))
    names = ("round1", "round2", "round3_quotient", "round3_commit", "round4", "round5")
    return {k: arr[i] for i, k in enumerate(names)}


def prove_raw(ctx: Context, pk: ProvingKey, wires_ptr: int, pub_inputs: np.ndarray, blinders: np.ndarray) -> B200Proof:
    """prove with the wire table given by address (pinned host or device memory)."""
    p = _table_proof(pk, wires_ptr, pub_inputs, blinders, "prove_raw")
    _lib.check(ctx._lib.b200_plonk_prove(ctx._h, pk._h, p.src, _opt(p.pub), _ptr(p.bl), C.byref(p.proof), None, None))
    return p.proof


class B200LinkProof(_lib.STRUCTS["b200_link_proof"]):
    """b200_link_proof: mpc-plonk `LinkingProof { quotient_commitment, opening_proof }`."""

    def to_array(self) -> np.ndarray:
        return np.frombuffer(bytes(self), dtype=np.uint64).copy()


@dataclass
class GroupLayout:
    """mpc-relation `GroupLayout`: the link group occupies the roots g^(offset + i), i < size,
    of the 2^alignment-th roots of unity."""
    alignment: int
    offset: int
    size: int


def link_proofs(ctx: Context, srs: Bases, hint_a: LinkingHint, hint_b: LinkingHint, layout: GroupLayout):
    """`PlonkKzgSnark::link_proofs::<SolidityTranscript>` (proof_linking/intent_only.rs:42-47).
    Returns (B200LinkProof, eta)."""
    it, keep = _link_item(hint_a, hint_b, layout, len(srs), "link_proofs: the link")
    _lib.check(ctx._lib.b200_plonk_link(ctx._h, srs._h, it.a1, it.len1, it.a2, it.len2, it.comm1, it.comm2, it.alignment,
                                        it.offset, it.size, it.proof, it.eta))
    return keep[4], keep[5]


B200LinkItem = _lib.STRUCTS["b200_link_item"]  # one link proof of a batch


def _link_item(hint_a, hint_b, lay, srs_len: int, where: str):
    """One link proof of hint_a to hint_b on `lay`, checked: (its b200_link_item, (a1, a2, c1, c2, proof, eta)): the
    arrays the item points into, then the buffers it writes."""
    p1, n1, a1, c1 = _link_hint(hint_a, where, "hint_a")
    p2, n2, a2, c2 = _link_hint(hint_b, where, "hint_b")
    _check_layout(lay, max(n1, n2), srs_len, where)
    proof, eta = B200LinkProof(), np.zeros(4, dtype=np.uint64)
    item = B200LinkItem(p1, n1, p2, n2, _ptr(c1), _ptr(c2), lay.alignment, lay.offset, lay.size,
                        C.cast(C.pointer(proof), C.c_void_p), _ptr(eta))
    return item, (a1, a2, c1, c2, proof, eta)


def _link_items(srs: Bases, triples, where: str = "link_proofs_batch"):
    """A link batch: (its b200_link_item array, each item's arrays and buffers as `_link_item` gives them)."""
    triples, srs_len = list(triples), len(srs)
    built = []
    for i, t in enumerate(triples):
        if len(t) != 3:
            raise ValueError(f"{where}: item {i} is not a (hint_a, hint_b, layout) triple")
        built.append(_link_item(*t, srs_len, f"{where}: item {i}"))
    return (B200LinkItem * max(1, len(built)))(*(it for it, _ in built)), [keep for _, keep in built]


def _link_batch_results(keep, statuses):
    st = [int(statuses[i]) for i in range(len(keep))]
    return [x[4] for x in keep], [x[5] if s == _lib.B200_OK else None for x, s in zip(keep, st)], st


def link_proofs_batch(ctx: Context, srs: Bases, triples):
    """`link_proofs` for many (hint_a, hint_b, layout) triples in ONE call (`b200_plonk_link_batch`).  A hint's
    linking_wire_poly is an array, or (address, length) of one in device or pinned host memory.  Returns
    (proofs, etas, statuses): item i's proof and eta equal `link_proofs` of the same triple; statuses[i] is 0, or -7
    (B200_ERR_UNSATISFIED) when the two polynomials differ on the group, in which case the proof is zeroed and the eta is
    None.  Argument errors raise ValueError before any device work; other failures raise B200Error."""
    items, keep = _link_items(srs, triples, "link_proofs_batch")
    k = len(keep)
    statuses = (C.c_int * max(1, k))()
    rc = ctx._lib.b200_plonk_link_batch(ctx._h, srs._h, items, k, statuses)
    if rc not in (_lib.B200_OK, _lib.B200_ERR_UNSATISFIED):
        _lib.check(rc)
    return _link_batch_results(keep, statuses)


SettlementLink = _lib.STRUCTS["b200_settlement_link"]  # one stored hint of a settlement and its group


def compute_poseidon_hash_batch(ctx: Context, values: np.ndarray) -> np.ndarray:
    """`batch` x `crypto::hash::compute_poseidon_hash(&values[i])` (crates/crypto/src/hash/mod.rs:12-18):
    values has shape (batch, len, 4) Montgomery; returns (batch, 4)."""
    v = np.ascontiguousarray(values, dtype=np.uint64)
    batch, ln = v.shape[0], v.shape[1]
    out = np.zeros((batch, 4), dtype=np.uint64)
    _lib.check(ctx._lib.b200_poseidon2_hash_batch(ctx._h, _ptr(v) if v.size else None, batch, ln, _ptr(out)))
    return out


def merkle_root_batch(ctx: Context, leaf_hashes: np.ndarray, sisters: np.ndarray, is_right: np.ndarray) -> np.ndarray:
    """Roots of a batch of Merkle openings (`b200_poseidon2_merkle_root_batch`): leaf_hashes (batch, 4), sisters
    (batch, height, 4) Montgomery limbs, is_right (batch, height) booleans -> (batch, 4)."""
    leaf = np.ascontiguousarray(leaf_hashes, dtype=np.uint64).reshape(-1, 4)
    batch = leaf.shape[0]
    sis = np.ascontiguousarray(sisters, dtype=np.uint64).reshape(batch, -1, 4)
    height = sis.shape[1]
    bits = np.ascontiguousarray(is_right, dtype=np.uint8).reshape(batch, height)
    out = np.zeros((batch, 4), dtype=np.uint64)
    _lib.check(ctx._lib.b200_poseidon2_merkle_root_batch(ctx._h, _ptr(leaf), _ptr(sis) if sis.size else None,
                                                         bits.ctypes.data_as(C.c_void_p) if bits.size else None, batch, height,
                                                         _ptr(out)))
    return out


def csprng_batch(ctx: Context, seeds: np.ndarray, first_index, count: int) -> np.ndarray:
    """`count` consecutive values of each Poseidon CSPRNG stream (`b200_poseidon2_csprng_batch`): seeds (batch, 4)
    Montgomery limbs, first_index (batch,) integers -> (batch, count, 4)."""
    sd = np.ascontiguousarray(seeds, dtype=np.uint64).reshape(-1, 4)
    idx = np.ascontiguousarray(first_index, dtype=np.uint64).reshape(-1)
    out = np.zeros((sd.shape[0], count, 4), dtype=np.uint64)
    _lib.check(ctx._lib.b200_poseidon2_csprng_batch(ctx._h, _ptr(sd), _ptr(idx), sd.shape[0], count, _ptr(out)))
    return out


def poseidon2_permute_batch(ctx: Context, states: np.ndarray) -> np.ndarray:
    """`Poseidon2Sponge::permute` (poseidon2.rs:90-110) on (batch, 3, 4) states; returns the permuted copy."""
    s = np.array(states, dtype=np.uint64, copy=True, order="C")
    _lib.check(ctx._lib.b200_poseidon2_permute_batch(ctx._h, _ptr(s), s.shape[0]))
    return s


# ---- names the reference gives these objects (circuit-types/src/lib.rs:72-101; SURVEY.md §8 row a11) ------------
PlonkProof = B200Proof                 # `pub type PlonkProof = Proof<SystemCurve>`
PlonkLinkProof = B200LinkProof         # `pub type PlonkLinkProof = LinkingProof<SystemCurve>`
ProofLinkingHint = LinkingHint         # `pub type ProofLinkingHint = LinkingHint<SystemCurve>`
ProverError = _lib.B200Error           # circuit-types/src/errors.rs:33-58: a failing prove surfaces as an error value


BundleProof = _lib.STRUCTS["b200_bundle_proof"]
BundleLink = _lib.STRUCTS["b200_bundle_link"]
BundleWitness = _lib.STRUCTS["b200_bundle_witness"]


def _bundle_links(links, n_proofs: int, where: str):
    """The b200_bundle_link array of a bundle and the link proofs it writes into; a link naming a proof outside the
    bundle raises ValueError before any device call."""
    arr_l = (BundleLink * max(len(links), 1))()
    out_links = []
    for i, (a, b, lay) in enumerate(links):
        if not (0 <= a < n_proofs and 0 <= b < n_proofs):
            raise ValueError(f"{where}: link {i} names proof ({a}, {b}) of a bundle of {n_proofs}")
        lp = B200LinkProof()
        arr_l[i].a, arr_l[i].b, arr_l[i].alignment, arr_l[i].offset, arr_l[i].size = a, b, lay.alignment, lay.offset, lay.size
        arr_l[i].proof = C.cast(C.pointer(lp), C.c_void_p)
        out_links.append(lp)
    return arr_l, out_links


@_prover_errors
def _bundle_job(proofs, links, resolve, build, struct, where: str):
    """A bundle: `proofs` = [(key, *inputs)], each proof made by build(key's shape, *inputs) (`_table_proof` or
    `_witness_proof`) into a `struct` entry; resolve(key) -> (C handle, shape).  Returns (entry array, link array, what the
    job reads, what `wait` returns: ([proofs], [link polys], [link proofs]), and [pub_inputs] for witnesses)."""
    ps, entries = [], []
    for i, (key, *inputs) in enumerate(proofs):
        h, shape = resolve(key)
        ps.append(build(shape, *inputs, f"{where}: proof {i}", link=True))
        entries.append(ps[-1].entry(h))
    arr_l, out_links = _bundle_links(links, len(ps), where)
    out = ([p.proof for p in ps], [p.link for p in ps], out_links)
    if struct is BundleWitness:
        out += ([p.pub for p in ps],)
    return (struct * max(1, len(ps)))(*entries), arr_l, (ps, [p[0] for p in proofs]), out


# ---- queued jobs of a pool or a box --------------------------------------------------------------------------------
# Each builder checks one job kind's arguments (ProverError or ValueError, before any library call) and returns
# (args, finish, held): the C arguments after the pool or box handle and, where the entry takes them, the SRS and the key
# handle (a single proof's args start at its key handle); finish(rc), which turns the job's status into what `wait`
# returns; and the objects the job reads until then.  A pool and a box submit the same job through their own entry point.

def _finish(results, batch: bool = False):
    """finish(rc) of a job: raises for a failed job, else returns results().  A batch job (`batch`) reports an unsatisfied
    or refused item in its statuses, so only its other failures raise."""
    def finish(rc):
        if not (batch and rc == _lib.B200_ERR_UNSATISFIED):
            _lib.check(rc)
        return results()
    return finish


@_prover_errors
def _prove_job(h, shape, build, *inputs, with_link_poly: bool, where: str):
    """One proof, made by build(shape, *inputs) (`_table_proof` or `_witness_proof`).  args are its pool entry's fields, key
    handle `h` first: the arguments of the single-proof submits.  `wait` returns the proof, or (proof, link_poly) with
    `with_link_poly`, with a witness proof's pub_inputs after them."""
    p = build(shape, *inputs, where, link=with_link_poly)
    e = p.entry(h)
    out = (p.proof,) + ((p.link,) if with_link_poly else ()) + ((p.pub,) if p.witness else ())
    return tuple(getattr(e, f) for f, _ in e._fields_), _finish(lambda: out if len(out) > 1 else out[0]), p


SettlementLink = _lib.STRUCTS["b200_settlement_link"]  # one stored hint of a settlement and its group


@_prover_errors
def _settlement_job(h, shape, srs_len, links, build, *inputs, where: str):
    """A settlement: the statement's proof made by build(shape, *inputs) (`_table_proof` or `_witness_proof`) in its pool
    entry, key handle `h`, and links = [(LinkingHint, GroupLayout)] from stored hints to the statement's own (srs_len None:
    the SRS length is not known here).  args start at a pointer to the entry.  `wait` returns (proof, link_proofs,
    statuses), with a witness settlement's pub_inputs after them, like `PlonkKzgSnark.prove_settlement[_witness]`."""
    p = build(shape, *inputs, where)
    links = list(links)
    arr = (SettlementLink * max(1, len(links)))()
    held, out = [], []
    for i, t in enumerate(links):
        if len(t) != 2:
            raise ValueError(f"{where}: link {i} is not a (hint, layout) pair")
        hint, lay = t
        ptr, n, a, c = _link_hint(hint, f"{where}: link {i}", "hint")
        _check_layout(lay, max(n, shape.domain_size + 2), srs_len, f"{where}: link {i}")
        lp = B200LinkProof()
        arr[i] = SettlementLink(ptr, n, _ptr(c), lay.alignment, lay.offset, lay.size, C.cast(C.pointer(lp), C.c_void_p), None)
        held += [a, c, hint]
        out.append(lp)
    st = (C.c_int * (len(out) + 1))()
    pub = (p.pub,) if p.witness else ()
    finish = _finish(lambda: (p.proof, out, list(st)) + pub, batch=True)
    return (C.pointer(p.entry(h)), arr, len(out), st), finish, (p, held)


def _verify_job(vks, pub_inputs, proofs, links, combined: bool, g2, where: str):
    """One verification job.  The C call copies every input, so only the outputs have to live until the wait, which
    returns what `verify_each` (a verdict list) or, `combined`, `batch_verify` ((all_ok, verdicts)) returns."""
    b = _VerifyBatch(vks, pub_inputs, proofs, links, g2, where)
    if not hasattr(b, "args"):  # no items and no G2 pair: a job still checks its G2 records
        raise ValueError("a verification job without items needs g2=(g2_h, g2_tau_h)")
    verdicts = (C.c_uint8 * max(1, b.n_c))()
    ok = C.c_int(0) if combined else None

    def results():
        v = b.verdicts(verdicts)
        return v if ok is None else (bool(ok.value) and len(b.c_proofs) == b.n_proofs, v)
    return (int(combined), *b.args, C.byref(ok) if combined else None, verdicts), _finish(results), ()


class _Tickets:
    """The tickets a pool or a box handed out and nobody has waited for yet: `_jobs` maps ticket -> (finish, held)."""

    def _submit(self, c_submit, args, finish, held) -> int:
        ticket = C.c_uint64()
        _lib.check(c_submit(self._h, *args, C.byref(ticket)))
        self._jobs[ticket.value] = (finish, held)
        return ticket.value

    def _wait(self, c_wait, ticket: int, *info):
        rc = c_wait(self._h, ticket, *info)
        finish, _ = self._jobs.pop(ticket, (None, None))
        if finish is None:  # not a ticket of this object
            _lib.check(rc)
            return None
        return finish(rc)

    def _expedite(self, c_expedite, ticket: int) -> int:
        moved = C.c_size_t()
        _lib.check(c_expedite(self._h, ticket, C.byref(moved)))
        return moved.value

    def _wait_info(self, c_wait_info, ticket: int):
        info = (C.c_uint64 * 2)()
        result = self._wait(c_wait_info, ticket, info)
        return result, int(info[0]), int(info[1])

    def _cancel(self, c_name: str, ticket: int) -> int:
        # the ticket keeps its buffers: a running job may write them until it reaches an abort point, so they live
        # until its wait
        ticket = _ticket(ticket, "cancel")
        dropped = C.c_size_t()
        _lib.check(getattr(self._lib, c_name)(self._h, ticket, C.byref(dropped)))
        return dropped.value

    def _cancel_all(self, c_cancel_all) -> int:
        dropped = C.c_size_t()
        _lib.check(c_cancel_all(self._h, C.byref(dropped)))
        return dropped.value


def _ticket(ticket, who: str) -> int:
    if isinstance(ticket, bool) or not isinstance(ticket, int) or not 0 < ticket < 1 << 64:
        raise ValueError(f"{who}: a ticket is an int in [1, 2^64), not {ticket!r}")
    return ticket


def _express_count(express, who: str) -> int:
    if isinstance(express, bool) or not isinstance(express, int) or express < 0:
        raise ValueError(f"{who}: the express worker count must be an int >= 0, not {express!r}")
    return express


def _express_sms(express_sms, express: int, who: str) -> int:
    """The reserved SM count of b200reserved.h, checked as the library checks it (0: no partition)."""
    if isinstance(express_sms, bool) or not isinstance(express_sms, int) or express_sms < 0:
        raise ValueError(f"{who}: express_sms must be an int >= 0, not {express_sms!r}")
    if express_sms and (express_sms % 8 or express_sms > 248):
        raise ValueError(f"{who}: express_sms must be a multiple of 8 in [8, 248], not {express_sms}")
    if express_sms and express == 0:
        raise ValueError(f"{who}: express_sms reserves SMs for express workers: it needs express >= 1")
    return express_sms


def _mask_sms(mask) -> set:
    return {64 * i + b for i, word in enumerate(mask) for b in range(64) if (int(word) >> b) & 1}


class ProverPool(_Tickets):
    """b200_pool: the device-side counterpart of the reference's `NativeProofManager` thread pool
    (crates/workers/proof-manager/src/implementations/native_proof_manager.rs:138-201, `spawn_fifo`
    per job).  `workers` proofs are in flight on one GPU; keys and SRS tables are shared.

    Buffers passed to `submit_*` are kept alive by the pool object until the ticket is waited for.

    `express` workers (b200express.h) take only jobs moved to the express queue by `expedite(ticket)`; their contexts'
    streams rank above the normal workers'.  Any pool can expedite: with no express workers the express queue is the
    front of the line.

    `express_sms` > 0 (b200reserved.h) also splits the device's SMs: the express workers run on a group of at least that
    many SMs (a multiple of 8), the normal workers on the rest, so that an expedited job's kernels never wait for the
    load's running blocks; `partition()` gives the two groups' sizes as the split rounded them."""

    def __init__(self, device: int = 0, workers: int = 6, express: int = 0, express_sms: int = 0):
        express = _express_count(express, "ProverPool")
        express_sms = _express_sms(express_sms, express, "ProverPool")
        self._lib = _lib.load()
        h = C.c_void_p()
        if express_sms:
            _lib.check(self._lib.b200_pool_create_reserved(device, workers, express, express_sms, C.byref(h)))
        else:
            _lib.check(self._lib.b200_pool_create_express(device, workers, express, C.byref(h)))
        self._h = h
        self.device = device
        self._jobs = {}
        self._borrowed = []

    @property
    def workers(self) -> int:
        return int(self._lib.b200_pool_workers(self._h))

    def partition(self):
        """(normal SMs, express SMs) of a pool made with `express_sms` (`b200_pool_partition`); (0, 0) without one."""
        out = (C.c_uint * 2)()
        _lib.check(self._lib.b200_pool_partition(self._h, out))
        return int(out[0]), int(out[1])

    def probe_sms(self, worker: int) -> set:
        """The SM ids a small kernel reached on each stream of worker `worker`'s context, eagerly and under graph replay
        (`b200_pool_probe_sms`; express workers after the normal ones)."""
        mask = (C.c_uint64 * 4)()
        _lib.check(self._lib.b200_pool_probe_sms(self._h, worker, mask))
        return _mask_sms(mask)

    def context(self, worker: int = 0) -> Context:
        """Worker `worker`'s context (borrowed: the pool frees it), for set-up calls."""
        raw = self._lib.b200_pool_ctx(self._h, worker)
        if not raw:
            raise IndexError("worker index out of range")
        ctx = Context.__new__(Context)
        ctx._lib, ctx._h, ctx.device, ctx._borrowed = self._lib, C.c_void_p(raw), self.device, True
        ctx.close = lambda: None  # the pool owns it
        self._borrowed.append(ctx)
        return ctx

    @staticmethod
    def _resolve(pk):
        return pk._h, pk

    def submit_prove(self, pk: "ProvingKey", wires_ptr: int, pub_inputs: np.ndarray, blinders: np.ndarray,
                     with_link_poly: bool = False, keep=None) -> int:
        """Queue one proof; returns the ticket.  `wires_ptr`: address of the 5 x n wire table (pinned host
        or device memory), which the caller keeps valid until `wait(ticket)` returns (pass the owning
        object as `keep` to let the pool hold a reference)."""
        args, finish, p = _prove_job(pk._h, pk, _table_proof, wires_ptr, pub_inputs, blinders,
                                     with_link_poly=with_link_poly, where="submit_prove")
        return self._submit(self._lib.b200_pool_submit_prove, args, finish, (p, keep, pk))

    def submit_prove_witness(self, pk: "ProvingKey", witness, blinders: np.ndarray, with_link_poly: bool = False,
                             keep=None) -> int:
        """Queue one proof from a witness vector (array, or address in pinned host or device memory kept valid until
        `wait(ticket)` returns) of a key made by `preprocess_wiring`; returns the ticket.  `wait(ticket)` returns
        (proof, pub_inputs), or (proof, link_poly, pub_inputs) with `with_link_poly`."""
        args, finish, p = _prove_job(pk._h, pk, _witness_proof, witness, blinders, with_link_poly=with_link_poly,
                                     where="submit_prove_witness")
        return self._submit(self._lib.b200_pool_submit_prove_witness, args, finish, (p, keep, pk))

    def submit_prove_batch(self, pk: "ProvingKey", wires_list, pub_inputs_list, blinders_list, link_hints: bool = False,
                           keep=None) -> int:
        """Queue one `b200_plonk_prove_batch` as a single job on one worker; returns the ticket.  Arguments as for
        `PlonkKzgSnark.prove_batch`; wire tables given by address stay owned by the caller until `wait(ticket)` returns
        (pass their owners as `keep`).  `wait(ticket)` returns (proofs, hints, statuses) like `prove_batch`."""
        items, ps = _prove_items(pk, wires_list, pub_inputs_list, blinders_list, link_hints, False, "submit_prove_batch")
        statuses = (C.c_int * max(1, len(ps)))()
        finish = _finish(lambda: _batch_results(ps, statuses, link_hints, False), batch=True)
        return self._submit(self._lib.b200_pool_submit_prove_batch, (pk._h, items, len(ps), statuses), finish,
                            (ps, keep, pk))

    def submit_link(self, srs: "Bases", hint_a: "LinkingHint", hint_b: "LinkingHint", layout: "GroupLayout") -> int:
        it, keep = _link_item(hint_a, hint_b, layout, len(srs), "submit_link: the link")
        args = (srs._h, it.a1, it.len1, it.a2, it.len2, it.comm1, it.comm2, it.alignment, it.offset, it.size, it.proof)
        return self._submit(self._lib.b200_pool_submit_link, args, _finish(lambda: keep[4]), (keep, srs))

    def submit_link_batch(self, srs: "Bases", triples, keep=None) -> int:
        """Queue one `b200_plonk_link_batch` as a single job on one worker; returns the ticket.  Arguments as for
        `link_proofs_batch`; polynomials given by address stay owned by the caller until `wait(ticket)` returns (pass
        their owners as `keep`).  `wait(ticket)` returns (proofs, etas, statuses) like `link_proofs_batch`."""
        items, held = _link_items(srs, triples, "submit_link_batch")
        statuses = (C.c_int * max(1, len(held)))()
        finish = _finish(lambda: _link_batch_results(held, statuses), batch=True)
        return self._submit(self._lib.b200_pool_submit_link_batch, (srs._h, items, len(held), statuses), finish,
                            (held, keep, srs))

    def submit_bundle(self, srs: "Bases", proofs, links) -> int:
        """One ticket for a whole proof bundle (`b200_pool_submit_bundle`): `proofs` = [(pk, wires_ptr, pub_inputs,
        blinders)], `links` = [(a, b, GroupLayout)] — link proof between the hints of proofs a and b, forked inside the
        pool once every proof is in (native_proof_manager.rs:526-584, 726-782).  `wait(ticket)` returns
        ([B200Proof], [link polys], [B200LinkProof])."""
        arr_p, arr_l, keep, out = _bundle_job(proofs, links, self._resolve, _table_proof, BundleProof, "submit_bundle")
        return self._submit(self._lib.b200_pool_submit_bundle, (srs._h, arr_p, len(proofs), arr_l, len(links)),
                            _finish(lambda: out), (keep, srs))

    def submit_bundle_witness(self, srs: "Bases", proofs, links) -> int:
        """`submit_bundle` with every proof given as a witness vector (`b200_pool_submit_bundle_witness`): `proofs` =
        [(pk, witness, blinders)], pk a key made by `preprocess_wiring`, witness an array or an address (pinned host or
        device memory, kept valid until `wait(ticket)` returns) as `submit_prove_witness` takes.  `wait(ticket)` returns
        ([B200Proof], [link polys], [B200LinkProof], [pub_inputs])."""
        arr_p, arr_l, keep, out = _bundle_job(proofs, links, self._resolve, _witness_proof, BundleWitness,
                                              "submit_bundle_witness")
        args = (srs._h if srs is not None else None, arr_p, len(proofs), arr_l, len(links))
        return self._submit(self._lib.b200_pool_submit_bundle_witness, args, _finish(lambda: out), (keep, srs))

    def submit_prove_witness_batch(self, pk: "ProvingKey", witnesses, blinders_list, link_hints: bool = False,
                                   keep=None) -> int:
        """Queue one `b200_plonk_prove_witness_batch` as a single job on one worker; returns the ticket.  Arguments as
        for `PlonkKzgSnark.prove_witness_batch`; witnesses given by address stay owned by the caller until `wait(ticket)`
        returns (pass their owners as `keep`).  `wait(ticket)` returns (proofs, hints, statuses, pub_inputs) like
        `prove_witness_batch`."""
        items, ps = _prover_errors(_witness_items)(pk, witnesses, blinders_list, link_hints, False,
                                                   "submit_prove_witness_batch")
        statuses = (C.c_int * max(1, len(ps)))()
        finish = _finish(lambda: _batch_results(ps, statuses, link_hints, False) + ([p.pub for p in ps],), batch=True)
        return self._submit(self._lib.b200_pool_submit_prove_witness_batch, (pk._h, items, len(ps), statuses), finish,
                            (ps, keep, pk))

    def submit_settlement(self, srs: "Bases", pk: "ProvingKey", wires, pub_inputs, blinders, links, keep=None) -> int:
        """Queue one `PlonkKzgSnark.prove_settlement` as ONE job on one worker (`b200_pool_submit_settlement`); returns the
        ticket.  Arguments as `prove_settlement` takes them; a wire table or hint given by address stays owned by the
        caller until `wait(ticket)` returns (pass its owner as `keep`).  `wait(ticket)` returns (proof, link_proofs,
        statuses) like `prove_settlement`."""
        args, finish, held = _settlement_job(pk._h, pk, len(srs), links, _table_proof, wires, pub_inputs, blinders,
                                             where="submit_settlement")
        return self._submit(self._lib.b200_pool_submit_settlement, (srs._h, *args), finish, (held, keep, pk, srs))

    def submit_settlement_witness(self, srs: "Bases", pk: "ProvingKey", witness, blinders, links, keep=None) -> int:
        """`submit_settlement` from the settlement's witness vector (`b200_pool_submit_settlement_witness`), arguments as
        `PlonkKzgSnark.prove_settlement_witness` takes them.  `wait(ticket)` returns (proof, link_proofs, statuses,
        pub_inputs)."""
        args, finish, held = _settlement_job(pk._h, pk, len(srs), links, _witness_proof, witness, blinders,
                                             where="submit_settlement_witness")
        return self._submit(self._lib.b200_pool_submit_settlement_witness, (srs._h, *args), finish, (held, keep, pk, srs))

    def submit_verify(self, vks, pub_inputs, proofs, links=(), combined: bool = False, g2=None) -> int:
        """Queue one verification job on some worker (`b200_pool_submit_verify`); returns the ticket.  Arguments as
        `PlonkKzgSnark.verify_each` / `.batch_verify` take them; every input is copied at submit.  `wait(ticket)` returns
        what `verify_each` returns (the verdict list), or with `combined` what `batch_verify` returns ((all_ok,
        verdicts): one combined pairing, the failing items found by bisection inside the job)."""
        job = _verify_job(vks, pub_inputs, proofs, links, combined, g2, "submit_verify")
        return self._submit(self._lib.b200_pool_submit_verify, *job)

    def wait(self, ticket: int):
        """Blocks until the job is done; returns its B200Proof (or (B200Proof, link_poly) when the job was
        submitted with `with_link_poly`, or the B200LinkProof of a link job); raises B200Error with the
        job's own status and message if it failed."""
        return self._wait(self._lib.b200_pool_wait, ticket)

    def expedite(self, ticket: int) -> int:
        """Move the ticket's queued jobs to the express queue (`b200_pool_expedite`); returns how many moved (0 once they
        have all started or finished, or when already expedited)."""
        return self._expedite(self._lib.b200_pool_expedite, ticket)

    def wait_info(self, ticket: int):
        """`wait` that also returns where and when the job finished (`b200_pool_wait_info`): (result, the pool's completed
        count right after the ticket's last job, the index of the worker that ran it — express workers after the normal
        ones)."""
        return self._wait_info(self._lib.b200_pool_wait_info, ticket)

    def cancel(self, ticket: int) -> int:
        """Cancel the ticket's job (`b200_pool_cancel`, b200cancel.h); returns how many of its queued jobs were dropped.
        Dropped jobs never run; a running one stops at its next abort point (a host round trip of the prover or the
        verifier).  `wait(ticket)` then raises B200Error with code B200_ERR_CANCELLED, or returns the job's result if it
        finished first.  A finished or already cancelled ticket drops 0."""
        return self._cancel("b200_pool_cancel", ticket)

    def cancel_all(self) -> int:
        """`cancel` for every job the pool holds (`b200_pool_cancel_all`); returns how many queued jobs were dropped.  Jobs
        submitted afterwards run as usual.  `cancel_all()` then `close()` stops the pool without draining its queue."""
        return self._cancel_all(self._lib.b200_pool_cancel_all)

    def wait_all(self) -> None:
        rc = self._lib.b200_pool_wait_all(self._h)
        self._jobs.clear()
        _lib.check(rc)

    def stats(self) -> dict:
        out = (C.c_uint64 * 4)()
        _lib.check(self._lib.b200_pool_stats(self._h, C.byref(out)))
        return dict(zip(("submitted", "completed", "failed", "queued"), (int(v) for v in out)))

    def close(self):
        if getattr(self, "_h", None):
            self._lib.b200_pool_destroy(self._h)
            self._h = None
            self._jobs.clear()
            for ctx in self._borrowed:  # their handles died with the pool
                ctx._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


@dataclass
class _BoxKeyShape:
    """What the box's Python side needs to know of a box key: output sizes and the witness length."""
    domain_size: int
    num_inputs: int
    num_vars: int


class ProverBox(_Tickets):
    """`b200_box`: every GPU of the box behind one object — one prover pool per device, the SRS tables and the proving
    keys replicated on each, jobs routed to the least-loaded device.  The single-process counterpart of running one
    `ProverPool` per rank under torchrun.  `express_per_device` express workers per device, and `express_sms` SMs
    reserved for them on every device, as in `ProverPool`."""

    def __init__(self, devices, workers_per_device: int = 6, express_per_device: int = 0, express_sms: int = 0):
        express_per_device = _express_count(express_per_device, "ProverBox")
        express_sms = _express_sms(express_sms, express_per_device, "ProverBox")
        self._lib = _lib.load()
        arr = (C.c_int * len(devices))(*devices)
        h = C.c_void_p()
        if express_sms:
            _lib.check(self._lib.b200_box_create_reserved(arr, len(devices), workers_per_device, express_per_device, express_sms,
                                                          C.byref(h)))
        else:
            _lib.check(self._lib.b200_box_create_express(arr, len(devices), workers_per_device, express_per_device, C.byref(h)))
        self._h, self._jobs, self.devices = h, {}, list(devices)
        self._shapes = {}  # key handle -> _BoxKeyShape, for the keys this box made

    def load_srs(self, points: np.ndarray, window_bits: int = 0, check_on_curve: bool = False):
        pts = np.ascontiguousarray(points, dtype=np.uint64).reshape(-1, 8)
        h = C.c_void_p()
        _lib.check(self._lib.b200_box_srs_load(self._h, _ptr(pts), pts.shape[0], window_bits, int(check_on_curve), C.byref(h)))
        return h

    def preprocess(self, srs, log_n: int, num_inputs: int, selectors: np.ndarray, perm: np.ndarray, k: np.ndarray):
        sel = np.ascontiguousarray(selectors, dtype=np.uint64).reshape(13, 1 << log_n, 4)
        pm = np.ascontiguousarray(perm, dtype=np.uint64).reshape(5 << log_n)
        kk = np.ascontiguousarray(k, dtype=np.uint64).reshape(5, 4)
        h = C.c_void_p()
        _lib.check(self._lib.b200_box_preprocess(self._h, srs, log_n, num_inputs, _ptr(sel), _ptr(pm), _ptr(kk), C.byref(h)))
        self._shapes[h.value] = _BoxKeyShape(1 << log_n, num_inputs, 0)
        return h

    def preprocess_wiring(self, srs, log_n: int, num_inputs: int, selectors: np.ndarray, wire_vars: np.ndarray, num_vars: int,
                          k: np.ndarray):
        """`PlonkKzgSnark.preprocess_wiring` on every device (`b200_box_preprocess_wiring`): a box key whose proofs are
        made from witness vectors."""
        sel = np.ascontiguousarray(selectors, dtype=np.uint64).reshape(13, 1 << log_n, 4)
        wv = np.ascontiguousarray(wire_vars, dtype=np.uint32).reshape(5 << log_n)
        kk = np.ascontiguousarray(k, dtype=np.uint64).reshape(5, 4)
        h = C.c_void_p()
        _lib.check(self._lib.b200_box_preprocess_wiring(self._h, srs, log_n, num_inputs, _ptr(sel), wv.ctypes.data_as(C.c_void_p),
                                                        num_vars, _ptr(kk), C.byref(h)))
        self._shapes[h.value] = _BoxKeyShape(1 << log_n, num_inputs, num_vars)
        return h

    def _resolve(self, pk):
        """(handle, shape) of a key this box made; ProverError for any other."""
        shape = self._shapes.get(getattr(pk, "value", pk))
        if shape is None:
            raise ProverError(_lib.B200_ERR_INVALID, "box: the key was not made by this box")
        return pk, shape

    def submit_prove(self, pk, wires_ptr: int, pub_inputs: np.ndarray, blinders: np.ndarray, with_link_poly: bool = False,
                     keep=None) -> int:
        """`ProverPool.submit_prove` on the least-loaded device (`b200_box_submit_prove`).  `wait(ticket)` returns the
        proof, or (proof, link_poly) with `with_link_poly`."""
        h, shape = self._resolve(pk)
        args, finish, p = _prove_job(h, shape, _table_proof, wires_ptr, pub_inputs, blinders,
                                     with_link_poly=with_link_poly, where="box.submit_prove")
        return self._submit(self._lib.b200_box_submit_prove, args, finish, (p, keep))

    def submit_prove_witness(self, pk, witness, blinders: np.ndarray, with_link_poly: bool = False, keep=None) -> int:
        """`ProverPool.submit_prove_witness` on the box (`b200_box_submit_prove_witness`): a witness in device memory runs
        on its own device, any other on the least-loaded one.  `wait(ticket)` returns (proof, pub_inputs), or (proof,
        link_poly, pub_inputs) with `with_link_poly`."""
        h, shape = self._resolve(pk)
        args, finish, p = _prove_job(h, shape, _witness_proof, witness, blinders, with_link_poly=with_link_poly,
                                     where="box.submit_prove_witness")
        return self._submit(self._lib.b200_box_submit_prove_witness, args, finish, (p, keep))

    def submit_bundle(self, srs, proofs, links) -> int:
        """`ProverPool.submit_bundle` on the least-loaded device (`b200_box_submit_bundle`): `proofs` = [(box key,
        wires_ptr, pub_inputs, blinders)].  `wait(ticket)` returns ([B200Proof], [link polys], [B200LinkProof])."""
        arr_p, arr_l, keep, out = _bundle_job(proofs, links, self._resolve, _table_proof, BundleProof, "box.submit_bundle")
        pks = (C.c_void_p * max(len(proofs), 1))(*[p[0] for p in proofs])
        return self._submit(self._lib.b200_box_submit_bundle, (srs, pks, arr_p, len(proofs), arr_l, len(links)),
                            _finish(lambda: out), keep)

    def submit_bundle_witness(self, srs, proofs, links) -> int:
        """`ProverPool.submit_bundle_witness` on one device of the box (`b200_box_submit_bundle_witness`): `proofs` = [(box
        key, witness, blinders)]; device-memory witnesses pin the bundle to their device (all on one).  `wait(ticket)`
        returns ([B200Proof], [link polys], [B200LinkProof], [pub_inputs])."""
        arr_p, arr_l, keep, out = _bundle_job(proofs, links, self._resolve, _witness_proof, BundleWitness,
                                              "box.submit_bundle_witness")
        pks = (C.c_void_p * max(len(proofs), 1))(*[p[0] for p in proofs])
        return self._submit(self._lib.b200_box_submit_bundle_witness, (srs, pks, arr_p, len(proofs), arr_l, len(links)),
                            _finish(lambda: out), keep)

    def submit_settlement(self, srs, pk, wires, pub_inputs, blinders, links, keep=None) -> int:
        """`ProverPool.submit_settlement` on one device of the box (`b200_box_submit_settlement`): pk a box key, srs a box
        SRS.  A wire table or hint polynomial in device memory pins the job to its device (all of them on one); otherwise
        the job goes to the least-loaded device.  `wait(ticket)` returns (proof, link_proofs, statuses)."""
        h, shape = self._resolve(pk)
        args, finish, held = _settlement_job(h, shape, None, links, _table_proof, wires, pub_inputs, blinders,
                                             where="box.submit_settlement")
        return self._submit(self._lib.b200_box_submit_settlement, (srs, h, *args), finish, (held, keep))

    def submit_settlement_witness(self, srs, pk, witness, blinders, links, keep=None) -> int:
        """`submit_settlement` from a witness vector (`b200_box_submit_settlement_witness`); the witness counts among the
        job's device pointers.  `wait(ticket)` returns (proof, link_proofs, statuses, pub_inputs)."""
        h, shape = self._resolve(pk)
        args, finish, held = _settlement_job(h, shape, None, links, _witness_proof, witness, blinders,
                                             where="box.submit_settlement_witness")
        return self._submit(self._lib.b200_box_submit_settlement_witness, (srs, h, *args), finish, (held, keep))

    def submit_verify(self, vks, pub_inputs, proofs, links=(), combined: bool = False, g2=None) -> int:
        """`ProverPool.submit_verify` on the least-loaded device (`b200_box_submit_verify`).  `wait(ticket)` returns the
        verdict list, or (all_ok, verdicts) with `combined`."""
        job = _verify_job(vks, pub_inputs, proofs, links, combined, g2, "box.submit_verify")
        return self._submit(self._lib.b200_box_submit_verify, *job)

    def verifying_key(self, pk):
        sel, sig = np.zeros((13, 8), dtype=np.uint64), np.zeros((5, 8), dtype=np.uint64)
        _lib.check(self._lib.b200_box_pk_verifying_key(pk, _ptr(sel), _ptr(sig)))
        return sel, sig

    def wait(self, ticket: int):
        return self._wait(self._lib.b200_box_wait, ticket)

    def expedite(self, ticket: int) -> int:
        """`ProverPool.expedite` on the pool of the ticket's device (`b200_box_expedite`)."""
        return self._expedite(self._lib.b200_box_expedite, ticket)

    def wait_info(self, ticket: int):
        """`ProverPool.wait_info` on the pool of the ticket's device (`b200_box_wait_info`)."""
        return self._wait_info(self._lib.b200_box_wait_info, ticket)

    def cancel(self, ticket: int) -> int:
        """`ProverPool.cancel` on the pool of the ticket's device (`b200_box_cancel`)."""
        return self._cancel("b200_box_cancel", ticket)

    def cancel_all(self) -> int:
        """`ProverPool.cancel_all` on every device (`b200_box_cancel_all`); returns the total dropped."""
        return self._cancel_all(self._lib.b200_box_cancel_all)

    def ticket_device(self, ticket: int) -> int:
        return self._lib.b200_box_ticket_device(self._h, ticket)

    def free_pk(self, pk):
        self._lib.b200_box_pk_free(self._h, pk)
        self._shapes.pop(getattr(pk, "value", pk), None)

    def free_srs(self, srs):
        self._lib.b200_box_srs_free(self._h, srs)

    def close(self):
        if getattr(self, "_h", None):
            self._lib.b200_box_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
