/* libb200prover — C ABI of the H100-native (sm_90a) proving backend for the PlonK prover behind
 * renegade-fi/renegade's crates/circuits.
 *
 * This is the drop-in boundary (SURVEY.md §8(b)).  The reference has no FFI for this path: its
 * prover calls Rust crates directly.  Each entry point below names the Rust call it replaces;
 * INTEGRATION.md shows the `extern "C"` block and the safe wrappers a maintainer adds in a new
 * `gpu-prover` shim crate (the existing crates deny `unsafe`: circuit-types/src/lib.rs:4).
 *
 * Conventions
 *   - plain pointers and sizes only; every handle is opaque and owned by the library;
 *   - caller owns all host buffers; the library never keeps a caller pointer past return;
 *   - return 0 on success, negative B200_ERR_* otherwise; never throws, never aborts;
 *     b200_last_error() returns a thread-local message for the last failure;
 *   - field element = 4 x uint64 little-endian limbs (32 bytes).  "Montgomery" = a * 2^256 mod p,
 *     exactly ark-ff's in-memory `Fp256<MontBackend>`; "canonical" = ark-ff `BigInt<4>`;
 *   - G1 affine point = x || y, 64 bytes, Montgomery — one record of the reference's SRS file
 *     (crates/circuits/circuit-types/src/primitives/srs.rs:172-182) and the payload of
 *     `Commitment(G1Affine)`; the identity is flagged separately (and stored as 64 zero bytes);
 *   - a context serialises the calls made on it; use one context per worker thread (rayon
 *     workers in native_proof_manager.rs:187-192) or per GPU for concurrency.
 *   - there is no CPU fallback: without a CUDA device every entry point fails with
 *     B200_ERR_NO_DEVICE.
 */
#ifndef B200PROVER_H
#define B200PROVER_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200_OK 0
#define B200_ERR_INVALID (-1)      /* bad argument */
#define B200_ERR_CUDA (-2)         /* CUDA runtime failure (message has the call) */
#define B200_ERR_NOMEM (-3)
#define B200_ERR_FORMAT (-4)       /* malformed .ptau */
#define B200_ERR_NOT_ON_CURVE (-5) /* srs.rs:179 "point not on curve" */
#define B200_ERR_NO_DEVICE (-6)
#define B200_ERR_UNSATISFIED (-7)  /* PlonkError::WrongQuotientPolyDegree: witness does not satisfy the circuit */

typedef struct b200_ctx b200_ctx;     /* one CUDA device + stream + scratch */
typedef struct b200_bases b200_bases; /* device-resident G1 bases + window tables (the SRS) */
typedef struct b200_pk b200_pk;       /* device-resident proving key of one circuit */

/* Flat proof, same field order as the reference's `PlonkProof` / `PlonkProofEvaluations`
 * (crates/relayer-types/types-proofs/src/rkyv_impls/plonk_proof_def.rs:168-222); commitments
 * are affine x||y Montgomery, evaluations Montgomery Fr; plookup_proof is always None. */
typedef struct {
    uint64_t wires_poly_comms[5][8];
    uint64_t prod_perm_poly_comm[8];
    uint64_t split_quot_poly_comms[5][8];
    uint64_t opening_proof[8];
    uint64_t shifted_opening_proof[8];
    uint64_t wires_evals[5][4];
    uint64_t wire_sigma_evals[4][4];
    uint64_t perm_next_eval[4];
} b200_proof;

/* ---- lifecycle ------------------------------------------------------------------------- */
/* device: CUDA ordinal.  Replaces nothing in the reference (it has no device). */
int b200_init(int device, b200_ctx** out);
void b200_shutdown(b200_ctx* ctx);
const char* b200_last_error(void);
/* "libb200prover <version> sm_90a" */
const char* b200_version(void);
/* Kernels launched by the library in this process so far (all contexts, all threads). */
uint64_t b200_kernel_launches(void);
/* Host time, in nanoseconds, the calling threads spent submitting those launches (sum over threads). */
uint64_t b200_launch_host_ns(void);
/* From the second proof of a key on a context, b200_plonk_prove replays each prover round as ONE CUDA graph (same kernels,
 * same order, same bytes out; b200_kernel_launches keeps counting the kernels executed).  b200_graph_launches: graph
 * submissions so far.  b200_ctx_use_graphs(ctx, 0) switches the replay off for a context (default: on, or B200_GRAPHS=0
 * in the environment). */
uint64_t b200_graph_launches(void);
int b200_ctx_use_graphs(b200_ctx* ctx, int on);

/* ---- SRS ------------------------------------------------------------------------------- */
/* Replaces parse_ptau_file / read_ptau_header / read_ptau_section1 / read_ptau_section2
 * (srs.rs:63-141): validates magic "ptau", version 1, 11 sections, the Fq modulus and
 * power >= 17, and returns a pointer INTO `bytes` to the first G1 record and the number of
 * records available in section 2.  Host-only, no device work. */
int b200_srs_parse_ptau(const uint8_t* bytes, size_t len, const uint8_t** g1_records,
                        size_t* n_records);

/* Uploads n affine points (64-byte records) and precomputes their window tables.
 * Replaces building `UnivariateUniversalParams.powers_of_g` (srs.rs:70) / the `commit_key`
 * held by `ProvingKey` (traits.rs:850).  window_bits = 0 lets the library choose the Pippenger window
 * for THROUGHPUT (several MSMs / proofs in flight on the GPU, the prover pool's regime: least multiplier
 * work), 1 for LATENCY (one MSM at a time: shortest dependent chains; e.g. c = 16 instead of 15 at 2^13
 * points), 8..23 fixes it.  The result does not depend on the window.
 * check_on_curve != 0 repeats the reference's `is_on_curve` assertion (srs.rs:178-179) on the
 * device and fails with B200_ERR_NOT_ON_CURVE (a coordinate >= q counts as off the curve). */
int b200_bases_load(b200_ctx* ctx, const uint8_t* points64, size_t n, int window_bits,
                    int check_on_curve, b200_bases** out);
/* Same, from points already in device memory (device pointer). */
int b200_bases_load_device(b200_ctx* ctx, const void* d_points64, size_t n, int window_bits,
                           b200_bases** out);
void b200_bases_free(b200_ctx* ctx, b200_bases* bases);
size_t b200_bases_len(const b200_bases* bases);
/* plan[0..3] = window bits c, digits per scalar, physical bucket windows, precomputed tables */
void b200_bases_plan(const b200_bases* bases, int plan[4]);

/* Replaces read_ptau_section3 (srs.rs:147-157): the first two G2 records of the section that follows section 2
 * (located by section 2's declared size, as the reference seeks to its end): h = tau^0 H, beta_h = tau^1 H, 128-byte
 * records x0||x1||y0||y1 Montgomery, the layout every verifier here takes.  Header checks as b200_srs_parse_ptau.
 * B200_ERR_FORMAT (b200_last_error says which) for a file that ends before section 3's two records, a section number
 * other than 3, a section 3 declared shorter than the two records, or a section 2 size that would leave the buffer;
 * B200_ERR_NOT_ON_CURVE for a record off the twist (a coordinate >= q included).  Host only. */
int b200_srs_parse_ptau_g2(const uint8_t* bytes, size_t len, uint64_t g2_h[16], uint64_t g2_tau_h[16]);

/* *in_subgroup = [ Q is a point of the twist of order r ] ([r]Q == O; the identity counts as not in the subgroup).
 * B200_ERR_NOT_ON_CURVE off the twist.  Host only. */
int b200_g2_in_subgroup(const uint64_t rec[16], int* in_subgroup);

typedef struct {
    uint64_t consistent;     /* 1: the combined check passed, e(sum rho^i P_i, tau H) == e(sum rho^i P_{i+1}, H), i < n-1 */
    uint64_t g1_generator;   /* P_0 == (1, 2), the G the verifiers use */
    uint64_t g2_subgroup;    /* h and beta_h both of order r */
    uint64_t n_bad;          /* with locate and consistent == 0: number of failing pairs (P_i, P_{i+1}); else 0 */
    uint64_t bad[8];         /* the first min(n_bad, 8) failing pair indices i, ascending */
} b200_srs_report;

/* Checks the first n powers of a loaded SRS against the G2 pair: that they are P_i = tau^i P_0 for the tau of
 * beta_h = tau h.  rho = keccak256("b200 srs check v1" || seed[32] || n as u64 big-endian || g2_h || g2_tau_h) read
 * big-endian mod r (1 if 0); the two weight vectors rho^i are filled on the device, both sums are one batch-2 MSM over
 * the resident bases on the context's stream (counted by b200_msm_timing_totals), and the pairing runs on the host.
 * The seed must be unknown to whoever made the file; then an inconsistent SRS passes with probability at most n / r.
 * With locate != 0 and a failed combined check, every consecutive pair e(P_i, tau H) == e(P_{i+1}, H) is checked on its
 * own on the device, one thread per pair, and n_bad / bad are filled (an off-curve point fails the pairs it is in).
 * The SRS is valid exactly when consistent && g1_generator && g2_subgroup.
 * B200_ERR_INVALID: NULL ctx / srs / g2 / seed / out, n == 0 or n > b200_bases_len(srs).  B200_ERR_NOT_ON_CURVE for a G2
 * record off the twist.  n == 1 checks the generator and the subgroup only (consistent = 1). */
int b200_srs_check(b200_ctx* ctx, const b200_bases* srs, size_t n, const uint64_t g2_h[16], const uint64_t g2_tau_h[16],
                   const uint8_t seed[32], int locate, b200_srs_report* out);

/* ---- MSM ------------------------------------------------------------------------------- */
/* out = sum_{i<n} scalars[i] * bases[base_off + i].
 * Replaces `VariableBaseMSM::msm_bigint(&bases[..], &scalars[..])` followed by
 * `.into_affine()` as used by jf-primitives `UnivariateKzgPCS::commit` (reached from
 * traits.rs:850,996; proof_linking/intent_only.rs:42-47).  scalars_montgomery = 0: canonical
 * `BigInt<4>` (what msm_bigint takes); 1: Montgomery `Fr` coefficients (what `commit` is
 * handed) — the conversion is fused into digit extraction.  Scalars must be < r. */
int b200_msm(b200_ctx* ctx, const b200_bases* bases, size_t base_off, const uint64_t* scalars,
             size_t n, int scalars_montgomery, uint64_t out_xy[8], int* out_is_identity);
/* Same with the scalars already resident in device memory (device pointer). */
int b200_msm_device(b200_ctx* ctx, const b200_bases* bases, size_t base_off,
                    const void* d_scalars, size_t n, int scalars_montgomery, uint64_t out_xy[8],
                    int* out_is_identity);

/* `batch` MSMs over the same bases in one pass: scalar vector i starts at d_scalars + i*stride
 * (elements), each of n scalars; out_xy receives batch x 64 bytes.  Replaces jf-primitives
 * `UnivariateKzgPCS::batch_commit` (the 5 wire / 5 quotient commitments of a proof). */
int b200_msm_batch_device(b200_ctx* ctx, const b200_bases* bases, size_t base_off,
                          const void* d_scalars, size_t n, size_t stride, unsigned batch,
                          int scalars_montgomery, uint64_t* out_xy, int* out_is_identity);

/* Kept for ABI compatibility, no effect: round 1's running-sum bucket reduction had a latency and a
 * throughput setting; the row/column tree reduction that replaced it has one shape for both uses. */
int b200_msm_tuning(b200_ctx* ctx, int throughput_mode);
/* Device-side phase timing (CUDA events recorded on the context's stream).  enable != 0 turns
 * it on for subsequent MSM calls, the batch provers' commitments included; out_ms (may be NULL)
 * receives the last single call's (b200_msm*, b200_plonk_prove, b200_plonk_link)
 * {total, sort = count+scan+scatter, bucket accumulation, bucket reduction} in ms. */
int b200_msm_timing(b200_ctx* ctx, int enable, float out_ms[4]);

/* Running totals of the bucket-accumulation kernel since the last reset while timing is enabled:
 * out = {milliseconds, (point, scalar) pairs, launches}, every MSM call on this context included
 * (the prover's batched commitments too, b200_plonk_prove_batch's and b200_plonk_link_batch's
 * included).  A proof of domain size n adds 4 launches and 13n + 32 pairs. */
int b200_msm_timing_totals(b200_ctx* ctx, int reset, double out[3]);

/* Sum of k affine points on the host (combining per-GPU partial MSM results after the NCCL
 * gather; ark-ec `Projective += Affine`). */
int b200_g1_sum_affine(const uint64_t* points_xy, const int* is_identity, size_t k,
                       uint64_t out_xy[8], int* out_is_identity);

/* ---- NTT ------------------------------------------------------------------------------- */
/* In-place transform of n = 2^log_n Montgomery Fr elements, natural order in and out.
 * Replaces Radix2EvaluationDomain::<Fr>::{fft_in_place, ifft_in_place, coset_fft_in_place,
 * coset_ifft_in_place} (ark-poly 0.4.2; coset shift = Fr::GENERATOR = 5; ifft scales by n^-1). */
int b200_ntt(b200_ctx* ctx, uint64_t* data, unsigned log_n, int inverse, int coset);
/* `batch` transforms `stride` elements apart, data in device memory (device pointer). */
int b200_ntt_device(b200_ctx* ctx, void* d_data, unsigned log_n, int inverse, int coset,
                    unsigned batch, size_t stride);
/* Device time (CUDA events around the kernels) of the last b200_ntt_device call, in ms. */
int b200_ntt_last_ms(b200_ctx* ctx, float* out_ms);
/* Radix2EvaluationDomain::group_gen (Montgomery). */
int b200_domain_generator(b200_ctx* ctx, unsigned log_n, uint64_t out[4]);

/* ---- synthetic inputs for benchmarks / parity tests (SURVEY.md §8(d)) ------------------- */
/* element i = SplitMix64(seed) outputs 4i..4i+3 as LE limbs, reduced mod r */
int b200_splitmix_fr_device(b200_ctx* ctx, uint64_t seed, size_t first, size_t n, int montgomery,
                            void* d_out);
/* known-discrete-log bases P_i = a_i * G, a_i = splitmix_fr(seed)[first + i]; 64 B records */
int b200_known_dlog_bases_device(b200_ctx* ctx, uint64_t seed, size_t first, size_t n,
                                 void* d_out);

/* ---- TurboPlonk prover (boundary B2, SURVEY.md §8(b)) ------------------------------------ */
/* Replaces `PlonkKzgSnark::<Bn254>::preprocess(&SYSTEM_SRS, &cs)` (traits.rs:850).
 * The host (Rust: `cs` after finalize_for_arithmetization) hands over the circuit structure:
 *   selectors_evals  13 x n selector values over the domain, column order
 *                    q_lc[0..4] q_mul[0..2] q_hash[0..4] q_o q_c q_ecc (Montgomery);
 *   perm             5n entries: perm[i*n + j] = i'*n + j', the copy-constraint permutation
 *                    over wire positions (column i, row j);
 *   k                the 5 coset representatives `vk.k` (Montgomery);
 *   num_inputs       public-input gates occupy rows 0..num_inputs-1.
 * Selector / sigma polynomials, their commitments (the VerifyingKey contents) and the coset
 * evaluations the quotient needs stay resident on the device.  srs must hold >= n + 3 points. */
int b200_plonk_preprocess(b200_ctx* ctx, const b200_bases* srs, unsigned log_n, size_t num_inputs,
                          const uint64_t* selectors_evals, const uint64_t* perm, const uint64_t* k,
                          b200_pk** out);
/* b200_plonk_preprocess from the circuit's wiring (`PlonkCircuit::wire_variables` after finalize_for_arithmetization)
 * instead of the permutation derived from it:
 *   wire_vars   5 x n variable indices (32 bits each), wire_vars[i*n + j] = the variable on wire i of row j, each < num_vars;
 *   num_vars    length of the witness vector a proof of this key takes (1 <= num_vars < 2^32).
 * The copy permutation is derived on the device: the positions p = i*n + j of one variable, in ascending p, form one
 * cycle, each mapped to the next and the last to the first (a variable used once maps to itself; variable numbers no
 * position uses are allowed).  The key is the key b200_plonk_preprocess builds from that permutation (same verifying key)
 * and additionally keeps wire_vars resident (20n bytes), so that proofs can be made from witness vectors
 * (b200_plonk_prove_witness).  Public input j is the witness value of the variable on the output wire (wire 4) of row j,
 * j < num_inputs: the public-input gates constrain w4 = public input.
 * B200_ERR_INVALID for an index >= num_vars (b200_last_error names the first such position) and for num_vars outside
 * [1, 2^32).  The grouping is a radix sort (CUB); its launches are not counted by b200_kernel_launches. */
int b200_plonk_preprocess_wiring(b200_ctx* ctx, const b200_bases* srs, unsigned log_n, size_t num_inputs,
                                 const uint64_t* selectors_evals, const unsigned* wire_vars, size_t num_vars,
                                 const uint64_t* k, b200_pk** out);
/* Length of the witness vector of a key made by b200_plonk_preprocess_wiring; 0 for a key made by b200_plonk_preprocess. */
size_t b200_pk_num_vars(const b200_pk* pk);
/* VerifyingKey commitments: 13 selector + 5 sigma commitments, 64 B each. */
int b200_pk_verifying_key(const b200_pk* pk, uint64_t* selector_comms, uint64_t* sigma_comms);
/* Shape of a key: number of public inputs and log2 of the domain size it was preprocessed for. */
size_t b200_pk_num_inputs(const b200_pk* pk);
unsigned b200_pk_log_n(const b200_pk* pk);
void b200_pk_free(b200_ctx* ctx, b200_pk* pk);

/* Replaces `PlonkKzgSnark::prove_with_link_hint::<_, _, SolidityTranscript>(&mut rng, &circuit,
 * &pk)` (traits.rs:996).  wires: 5 x n wire values (the witness table after synthesis; host
 * or device pointer);
 * pub_inputs: num_inputs values; blinders: the 17 Fr elements the reference draws from its RNG
 * (2 per wire polynomial, 3 for the permutation product, 4 for the quotient split), in draw
 * order, supplied by the caller so both sides can be made deterministic (SURVEY.md §0.3).
 * link_poly (may be NULL): the (n + 2)-coefficient blinded wire-0 polynomial of
 * `LinkingHint.linking_wire_poly`; its commitment is proof->wires_poly_comms[0].
 * challenges (may be NULL): beta, gamma, alpha, zeta, v, u for audit.
 * Fails with B200_ERR_UNSATISFIED where the reference returns WrongQuotientPolyDegree. */
int b200_plonk_prove(b200_ctx* ctx, const b200_pk* pk, const uint64_t* wires,
                     const uint64_t* pub_inputs, const uint64_t* blinders, b200_proof* proof,
                     uint64_t* link_poly, uint64_t* challenges);

/* b200_plonk_prove from the witness vector (`PlonkCircuit::witness`: num_vars x 4 limbs, Montgomery, host or device
 * pointer) of a key made by b200_plonk_preprocess_wiring.  The wire table is gathered on the device from the key's
 * resident wiring, so a proof uploads num_vars x 32 bytes instead of 5n x 32 and the host never builds the table.
 * proof, link_poly and challenges are byte-identical to b200_plonk_prove on the expanded table
 * wires[i*n + j] = witness[wire_vars[i*n + j]] with the public inputs read from the witness.
 * pub_inputs_out (may be NULL) receives the key's num_inputs public inputs.  A device witness (read in place when it is
 * 16-byte aligned) costs one extra stream synchronisation: its public inputs are read back before the transcript starts.
 * B200_ERR_INVALID for a key without wiring or a NULL ctx / pk / witness / blinders / proof. */
int b200_plonk_prove_witness(b200_ctx* ctx, const b200_pk* pk, const uint64_t* witness, const uint64_t* blinders,
                             b200_proof* proof, uint64_t* link_poly, uint64_t* challenges, uint64_t* pub_inputs_out);

/* One witness of a batch: the arguments of b200_plonk_prove. */
typedef struct {
    const uint64_t* wires;      /* 5 x n, host or device pointer */
    const uint64_t* pub_inputs; /* the key's num_inputs values */
    const uint64_t* blinders;   /* 17, draw order as b200_plonk_prove */
    b200_proof* proof;
    uint64_t* link_poly;        /* may be NULL; (n + 2) x 4 limbs */
    uint64_t* challenges;       /* may be NULL; beta gamma alpha zeta v u */
} b200_prove_item;
/* Proves k witnesses of ONE key together: every kernel launch covers all of them, every commitment round is one batched
 * MSM over the same SRS bases, and the five host round trips (Fiat–Shamir between rounds) are made once per batch.
 * Item i's proof, link_poly and challenges are byte-identical to b200_plonk_prove(ctx, pk, items[i].wires, ...).
 * statuses (may be NULL) receives k codes: B200_OK, or B200_ERR_UNSATISFIED for a witness that does not satisfy the
 * circuit (its proof is zeroed, its challenges are not written; every other item is still proved).  Returns B200_OK when
 * every item was proved, B200_ERR_UNSATISFIED when any was not; a CUDA, memory or argument error fails the whole call
 * (B200_ERR_INVALID for a NULL items pointer with k > 0, or an item with a NULL wires / blinders / proof pointer, or a NULL
 * pub_inputs for a key with num_inputs > 0).  k = 0 is accepted.
 * The batch runs in chunks of as many proofs as half the free device memory holds (about 100 MB per proof at n = 2^14,
 * 400 MB at 2^16; at most 64); the results do not depend on the chunk size.  A batch runs eagerly (no CUDA graphs) in
 * buffers of its own on the context, kept for the next batch: single proofs keep replaying their graphs. */
int b200_plonk_prove_batch(b200_ctx* ctx, const b200_pk* pk, const b200_prove_item* items, size_t k, int* statuses);

/* One witness vector of a batch: the arguments of b200_plonk_prove_witness. */
typedef struct {
    const uint64_t* witness;    /* num_vars x 4 limbs, host or device pointer */
    const uint64_t* blinders;   /* 17, draw order as b200_plonk_prove */
    b200_proof* proof;
    uint64_t* link_poly;        /* may be NULL; (n + 2) x 4 limbs */
    uint64_t* challenges;       /* may be NULL; beta gamma alpha zeta v u */
    uint64_t* pub_inputs_out;   /* may be NULL; the key's num_inputs values */
} b200_witness_item;
/* b200_plonk_prove_batch with the items given as witness vectors of a key made by b200_plonk_preprocess_wiring: one
 * launch gathers the wire tables of a whole chunk.  Item i's outputs are byte-identical to b200_plonk_prove_witness's;
 * statuses, return codes and chunking exactly as b200_plonk_prove_batch (B200_ERR_INVALID also for a key without wiring). */
int b200_plonk_prove_witness_batch(b200_ctx* ctx, const b200_pk* pk, const b200_witness_item* items, size_t k, int* statuses);

/* Flat link proof, field order of mpc-plonk `LinkingProof { quotient_commitment, opening_proof }`
 * (crates/relayer-types/types-proofs/src/mocks.rs:28-30). */
typedef struct {
    uint64_t quotient_commitment[8];
    uint64_t opening_proof[8];
} b200_link_proof;

/* Replaces `PlonkKzgSnark::link_proofs::<SolidityTranscript>(&hint_a, &hint_b, &group_layout,
 * &pk.commit_key)` (circuits-core/src/zk_circuits/proof_linking/intent_only.rs:42-47,
 * intent_and_balance.rs:66-72).  a1 / a2: the two `LinkingHint.linking_wire_poly` coefficient
 * vectors (Montgomery, host or device pointers; lengths may differ), comm1 / comm2 their
 * `linking_wire_comm`; (alignment, offset, size) = mpc-relation `GroupLayout`: the group sits on
 * the roots g^(offset + i), i < size, g the generator of the 2^alignment-th roots of unity.
 * eta (may be NULL) receives the Fiat–Shamir challenge.  Fails with B200_ERR_UNSATISFIED when a1 and a2
 * do not agree on the group (no link proof exists: wrong layout or mismatched witnesses); *proof is zeroed then and
 * eta is not written. */
int b200_plonk_link(b200_ctx* ctx, const b200_bases* srs, const uint64_t* a1, size_t len1,
                    const uint64_t* a2, size_t len2, const uint64_t* comm1, const uint64_t* comm2,
                    unsigned alignment, size_t offset, size_t size, b200_link_proof* proof,
                    uint64_t* eta);

/* One link proof of a batch: the arguments of b200_plonk_link. */
typedef struct {
    const uint64_t* a1; size_t len1;      /* host or device pointers, as b200_plonk_link */
    const uint64_t* a2; size_t len2;
    const uint64_t* comm1; const uint64_t* comm2;
    unsigned alignment; size_t offset; size_t size;
    b200_link_proof* proof;
    uint64_t* eta;                        /* may be NULL */
} b200_link_item;
/* Makes k link proofs together: the division by Z_D runs as one launch per step over all items of one transform size,
 * the k quotient commitments and the k opening proofs are one batched MSM each over the same SRS bases, and the host
 * derives every eta in one round trip.  Item i's proof and eta are byte-identical to b200_plonk_link(ctx, srs,
 * items[i].a1, ...); items may mix lengths, layouts and pointer kinds.
 * statuses (may be NULL) receives k codes: B200_OK, or B200_ERR_UNSATISFIED for an item whose a1 and a2 differ on the
 * group (its proof is zeroed, its eta is not written; every other item is still proved).  Returns B200_OK when every item
 * was proved, B200_ERR_UNSATISFIED when any was not.  An argument error fails the whole call before any device work with
 * B200_ERR_INVALID, and b200_last_error() names the item: a NULL ctx / srs, a NULL items pointer with k > 0, an item
 * with a NULL a1 / a2 / comm1 / comm2 / proof pointer, or one that b200_plonk_link refuses (size 0, size >= max(len1,
 * len2), alignment > 28, max(len1, len2) above the SRS length, or a transform above 2^28).  A CUDA or memory error fails
 * the whole call too.  k = 0 is accepted.
 * The batch runs in chunks of as many items as half the free device memory holds (at most 64); the results do not
 * depend on the chunk size.  It runs eagerly (no CUDA graphs) in the context's batch buffers, the ones
 * b200_plonk_prove_batch uses: single link proofs and single proofs keep replaying their graphs. */
int b200_plonk_link_batch(b200_ctx* ctx, const b200_bases* srs, const b200_link_item* items, size_t k, int* statuses);

/* ---- verification (host only; no device is needed or used) -----------------------------------
 * G2 points are 128-byte records x0 || x1 || y0 || y1 (Montgomery Fq), the layout of the ptau file's
 * G2 section read by srs.rs:185-199: g2_h = `UnivariateUniversalParams.h`, g2_tau_h = `.beta_h`.
 * *accepted = 1 / 0; a malformed proof element is a rejection, not an error.  Malformed: a G1 point off the curve,
 * or any field element outside [0, p) (a coordinate >= q; a public input, evaluation or vk.k >= r) — the
 * Montgomery limbs of a * 2^256 mod p are below p, so v + p is not another encoding of v.  A G2 record with a
 * coordinate >= q is off the curve: B200_ERR_NOT_ON_CURVE, here and in b200_pairing_check. */
/* Replaces `PlonkKzgSnark::<Bn254>::verify::<SolidityTranscript>(&vk, public_inputs, &proof, None)`
 * (traits.rs:1012-1018, reached from `SingleProverCircuit::verify`, traits.rs:1003-1019).  The
 * verifying key is passed flat: domain size 2^log_n, num_inputs, k[5], the 13 selector and 5 sigma
 * commitments (b200_pk_verifying_key). */
int b200_plonk_verify(unsigned log_n, size_t num_inputs, const uint64_t* k, const uint64_t* selector_comms,
                      const uint64_t* sigma_comms, const uint64_t* pub_inputs, const b200_proof* proof,
                      const uint64_t g2_h[16], const uint64_t g2_tau_h[16], int* accepted);
/* Replaces `PlonkKzgSnark::verify_link_proof::<SolidityTranscript>(&comm_a, &comm_b, &link_proof,
 * &group_layout, &open_key)` (proof_linking/intent_only.rs:77-84, `validate_*_link`). */
int b200_plonk_verify_link(const uint64_t* comm1, const uint64_t* comm2, unsigned alignment, size_t offset,
                           size_t size, const b200_link_proof* proof, const uint64_t g2_h[16],
                           const uint64_t g2_tau_h[16], int* accepted);
/* *is_one = [ prod_i e(P_i, Q_i) == 1 ] for k (G1, G2) pairs (64-byte / 128-byte records) with one
 * final exponentiation — the primitive under both verifiers and the reference's SRS unit test
 * (srs.rs:236-266: e(tau^i G, tau H) == e(tau^(i+1) G, H)). */
int b200_pairing_check(const uint64_t* g1_points, const uint64_t* g2_points, size_t k, int* is_one);

/* ---- batch verification (device) -------------------------------------------------------------
 * The flat verifying key b200_plonk_verify takes. */
typedef struct {
    unsigned log_n;
    size_t num_inputs;
    const uint64_t* k;              /* 5 x 4 */
    const uint64_t* selector_comms; /* 13 x 8 */
    const uint64_t* sigma_comms;    /* 5 x 8 */
} b200_verifying_key;
/* One proof of a batch: vks[vk] is its key; pub_inputs holds that key's num_inputs values. */
typedef struct {
    unsigned vk;
    const uint64_t* pub_inputs;
    const b200_proof* proof;
} b200_batch_proof;
/* One link proof of a batch: the arguments of b200_plonk_verify_link. */
typedef struct {
    const uint64_t* comm1;
    const uint64_t* comm2;
    unsigned alignment;
    size_t offset;
    size_t size;
    const b200_link_proof* proof;
} b200_batch_link;
/* Verifies n_proofs proofs and n_links link proofs with ONE pairing: every check e(A_i, [tau]_2) == e(B_i, [1]_2) is
 * weighted by a random rho_i and the sums are checked at once, e(sum rho_i A_i, [tau]_2) == e(sum rho_i B_i, [1]_2)
 * (two MSMs on the device, one pairing on the host).  The rho_i are Fiat–Shamir outputs over the whole batch:
 *   d_i   = keccak(0 || proof i's final transcript state), or
 *           keccak(1 || link i's final transcript state || pi || alignment u32 || offset u64 || size u64), big-endian;
 *   seed  = keccak("b200 batch verify v1" || d_0 || ... || d_{k-1} || g2_h || g2_tau_h);
 *   rho_i = keccak(seed || i as u64 big-endian) as a big-endian integer mod r (1 if that is 0).
 * Items are numbered proofs first, then links.  *all_accepted = 1 exactly when every item would be accepted by
 * b200_plonk_verify / b200_plonk_verify_link with the same G2 pair.  verdicts (may be NULL): n_proofs + n_links bytes,
 * verdicts[i] = that single verifier's answer for item i; when the combined check fails the failing items are found
 * by bisection over subsets (each step one MSM pair and one pairing).  With verdicts NULL the call stops after the
 * combined check.  An item with an off-curve G1 point or a field element outside [0, p) is rejected (verdict 0) and
 * left out of the combination.
 * Errors: B200_ERR_NOT_ON_CURVE for an off-curve G2 point (a coordinate >= q included); B200_ERR_INVALID for a vk
 * index out of range, log_n > 28, a link with alignment > 28 or size == 0, or a NULL pointer.  Zero items are
 * accepted. */
int b200_plonk_batch_verify(b200_ctx* ctx, const b200_verifying_key* vks, size_t n_vks, const b200_batch_proof* proofs,
                            size_t n_proofs, const b200_batch_link* links, size_t n_links, const uint64_t g2_h[16],
                            const uint64_t g2_tau_h[16], int* all_accepted, uint8_t* verdicts);
/* verdicts[i] (n_proofs + n_links bytes, proofs first) = b200_plonk_verify / b200_plonk_verify_link's answer for item i,
 * each item checked on its own, e(A_i, [tau]_2) == e(B_i, [1]_2), with no random combination and no bisection: the cost
 * does not depend on how many items fail.  The pairings run on the device, one thread per item.  Arguments, errors and
 * rejections of malformed items exactly as b200_plonk_batch_verify; verdicts may be NULL only when there are no items. */
int b200_plonk_verify_each(b200_ctx* ctx, const b200_verifying_key* vks, size_t n_vks, const b200_batch_proof* proofs,
                           size_t n_proofs, const b200_batch_link* links, size_t n_links, const uint64_t g2_h[16],
                           const uint64_t g2_tau_h[16], uint8_t* verdicts);
/* n_checks independent checks, all against the same m G2 points: is_one[c] = [ prod_{j<m} e(P_{c,j}, Q_j) == 1 ],
 * g1_points = n_checks x m 64-byte records (host), g2_points = m 128-byte records.  is_one[c] equals what
 * b200_pairing_check returns for check c's m pairs.  Where b200_pairing_check would fail for some check (a point off
 * the curve, a coordinate >= q), the call fails with the same code and b200_last_error() names the first such check
 * (an off-curve G2 point fails every check: the message names the point).  At most 8 pairs per check (m <= 8, else
 * B200_ERR_INVALID); m = 0 makes every check 1.  The G2 points are validated and their Miller-loop lines computed on
 * the host; the G1 checks, the Miller loops and the final exponentiations run on the device, one thread per check.
 * NULL pointers: B200_ERR_INVALID (g1_points / is_one may be NULL when there are no checks). */
int b200_pairing_check_many(b200_ctx* ctx, const uint64_t* g2_points, size_t m, const uint64_t* g1_points,
                            size_t n_checks, uint8_t* is_one);

/* Wall-clock milliseconds of the last proof's phases on this context: round 1, round 2, round 3
 * (coset NTTs + quotient + split), round 3 commitments, round 4, round 5, then two spare slots. */
int b200_plonk_last_timings(b200_ctx* ctx, float out_ms[8]);

/* ---- prover pool --------------------------------------------------------------------------
 * Device-side counterpart of the reference's `NativeProofManager` thread pool
 * (crates/workers/proof-manager/src/implementations/native_proof_manager.rs:138-201: jobs taken
 * from the queue are handed to rayon workers with `spawn_fifo`, one proof per worker): a FIFO
 * queue drained by `n_workers` host threads, each owning one context on `device`.  Proving keys
 * and SRS tables are shared read-only, so `n_workers` proofs are in flight on one GPU and the
 * latency-bound parts of one overlap the throughput-bound kernels of the others.
 * Ownership: `pub_inputs` and `blinders` are copied at submit; `wires`, the link polynomials and
 * every output buffer stay owned by the caller and must remain valid until the job's ticket has
 * been waited for.  Any thread may submit or wait. */
typedef struct b200_pool b200_pool;
int b200_pool_create(int device, unsigned n_workers, b200_pool** out);
/* Finishes the queued jobs, joins the workers, frees the contexts. */
void b200_pool_destroy(b200_pool* pool);
unsigned b200_pool_workers(const b200_pool* pool);
/* Worker i's context, for set-up calls (b200_bases_load, b200_plonk_preprocess) made while no job
 * is running; keys created on any context of the device can be used by every worker. */
b200_ctx* b200_pool_ctx(b200_pool* pool, unsigned worker);
/* Queue one `b200_plonk_prove(ctx_of_some_worker, pk, wires, pub_inputs, blinders, proof,
 * link_poly, NULL)`; *ticket identifies the job.  num_inputs must equal the key's
 * (b200_pk_num_inputs), else B200_ERR_INVALID. */
int b200_pool_submit_prove(b200_pool* pool, const b200_pk* pk, const uint64_t* wires,
                           const uint64_t* pub_inputs, size_t num_inputs, const uint64_t* blinders,
                           b200_proof* proof, uint64_t* link_poly, uint64_t* ticket);
/* Queue one `b200_plonk_prove_witness(ctx_of_some_worker, pk, witness, blinders, proof, link_poly, NULL, pub_inputs_out)`.
 * The blinders are copied at submit; the witness vector and the output buffers stay owned by the caller until the ticket
 * has been waited for.  B200_ERR_INVALID at submit for a NULL pool / pk / witness / blinders / proof / ticket or a key
 * without wiring. */
int b200_pool_submit_prove_witness(b200_pool* pool, const b200_pk* pk, const uint64_t* witness, const uint64_t* blinders,
                                   b200_proof* proof, uint64_t* link_poly, uint64_t* pub_inputs_out, uint64_t* ticket);
/* Queue one `b200_plonk_prove_batch(ctx_of_some_worker, pk, items, k, statuses)` as ONE job on one worker.  The items'
 * pub_inputs and blinders are copied at submit (the items array too); wires, the proof / link_poly / challenges buffers
 * and statuses (may be NULL) stay owned by the caller until the ticket has been waited for.  The ticket's status is the
 * call's: B200_ERR_UNSATISFIED when any item was not proved (see statuses). */
int b200_pool_submit_prove_batch(b200_pool* pool, const b200_pk* pk, const b200_prove_item* items, size_t k, int* statuses,
                                 uint64_t* ticket);
/* Queue one `b200_plonk_link(...)` (the reference forks its link proofs the same way:
 * native_proof_manager.rs:726-782). */
int b200_pool_submit_link(b200_pool* pool, const b200_bases* srs, const uint64_t* a1, size_t len1,
                          const uint64_t* a2, size_t len2, const uint64_t* comm1, const uint64_t* comm2,
                          unsigned alignment, size_t offset, size_t size, b200_link_proof* proof,
                          uint64_t* ticket);
/* Queue one `b200_plonk_link_batch(ctx_of_some_worker, srs, items, k, statuses)` as ONE job on one worker.  The items
 * array and each item's comm1 / comm2 are copied at submit; a1, a2, the proof and eta buffers and statuses (may be
 * NULL) stay owned by the caller until the ticket has been waited for.  A NULL pointer (pool, srs, ticket, items with
 * k > 0, or an item's a1 / a2 / comm1 / comm2 / proof) is refused at submit with B200_ERR_INVALID and nothing is queued.
 * The ticket's status is the call's: B200_ERR_UNSATISFIED when any item was refused (see statuses), B200_ERR_INVALID
 * for a bad layout or length. */
int b200_pool_submit_link_batch(b200_pool* pool, const b200_bases* srs, const b200_link_item* items, size_t k,
                                int* statuses, uint64_t* ticket);
/* One proof of a bundle, arguments as for b200_pool_submit_prove.  `link_poly` ((2^log_n + 2) x 4 limbs) is required
 * for every proof a link names. */
typedef struct {
    const b200_pk* pk;
    const uint64_t* wires;
    const uint64_t* pub_inputs;
    size_t num_inputs;
    const uint64_t* blinders;
    b200_proof* proof;
    uint64_t* link_poly;
} b200_bundle_proof;
/* One link proof of a bundle: `b200_plonk_link` between the hints of proofs[a] and proofs[b] (in that order) on the
 * group (alignment, offset, size). */
typedef struct {
    unsigned a;
    unsigned b;
    unsigned alignment;
    size_t offset;
    size_t size;
    b200_link_proof* proof;
} b200_bundle_link;
/* Queue a whole proof bundle under ONE ticket: the `n_proofs` proofs run through the pool; when all of them are in,
 * the `n_links` link proofs are forked onto the pool; the ticket completes after the last link proof (or with the
 * first failure).  A bundle links only proofs made inside it (e.g. 5 proofs + 4 links of one private match); a
 * settlement linked against hints kept from earlier validity proofs is b200_pool_submit_settlement
 * (b200settlement.h).  The arrays are copied at submit; the buffers they point to stay owned by the caller until the
 * ticket has been waited for. */
int b200_pool_submit_bundle(b200_pool* pool, const b200_bases* srs, const b200_bundle_proof* proofs, size_t n_proofs,
                            const b200_bundle_link* links, size_t n_links, uint64_t* ticket);
/* One proof of a bundle given as a witness vector, arguments as for b200_pool_submit_prove_witness: pk is a key made by
 * b200_plonk_preprocess_wiring, witness its num_vars x 4 limbs (host or device pointer).  `link_poly` ((2^log_n + 2) x 4
 * limbs) is required for every proof a link names; `pub_inputs_out` (may be NULL) receives the key's num_inputs values. */
typedef struct {
    const b200_pk* pk;
    const uint64_t* witness;
    const uint64_t* blinders;
    b200_proof* proof;
    uint64_t* link_poly;
    uint64_t* pub_inputs_out;
} b200_bundle_witness;
/* b200_pool_submit_bundle with the proofs given as witness vectors: each proof runs as one
 * b200_plonk_prove_witness on some worker; the links, the ticket and its status are exactly b200_pool_submit_bundle's
 * (links forked once every proof is in, first failure wins, an unsatisfied proof forks no links).  The arrays and the
 * blinders are copied at submit; the witness vectors and the output buffers stay owned by the caller until the ticket has
 * been waited for.  B200_ERR_INVALID at submit, with nothing queued, for a NULL pointer, a key without wiring
 * (b200_pk_num_vars == 0), or a link naming a missing proof or one without link_poly. */
int b200_pool_submit_bundle_witness(b200_pool* pool, const b200_bases* srs, const b200_bundle_witness* proofs,
                                    size_t n_proofs, const b200_bundle_link* links, size_t n_links, uint64_t* ticket);
/* Queue one `b200_plonk_prove_witness_batch(ctx_of_some_worker, pk, items, k, statuses)` as ONE job on one worker.  The
 * items array and each item's blinders are copied at submit; the witness vectors, the output buffers and statuses (may be
 * NULL) stay owned by the caller until the ticket has been waited for.  Refusals at submit, statuses and the ticket's
 * status as b200_pool_submit_prove_batch (B200_ERR_INVALID at submit also for a key without wiring). */
int b200_pool_submit_prove_witness_batch(b200_pool* pool, const b200_pk* pk, const b200_witness_item* items, size_t k,
                                         int* statuses, uint64_t* ticket);
/* Blocks until the job is done and returns ITS status (B200_OK or the error the prove/link call
 * returned; b200_last_error() of the waiting thread then holds the job's message).  A ticket can
 * be waited for once. */
int b200_pool_wait(b200_pool* pool, uint64_t ticket);
/* Blocks until the queue is empty and no job is running; returns the oldest failure among the
 * jobs not individually waited for (their tickets are consumed), else B200_OK. */
int b200_pool_wait_all(b200_pool* pool);
/* out = { submitted, completed, failed, queued } */
int b200_pool_stats(b200_pool* pool, uint64_t out[4]);

/* ---- all GPUs of a box behind one object: prover pools + replicated keys -----------------------
 * Whole proofs are independent jobs (SURVEY.md §8(e): replicas, one proof stream per GPU, no communication): a
 * `b200_box` holds one prover pool per device, `b200_box_srs_load` / `b200_box_preprocess` replicate the SRS tables and a
 * proving key on every device (identical results), and every job goes to the device with the fewest unfinished jobs.
 * What ONE host process — the relayer's `NativeProofManager` (native_proof_manager.rs:140-201) — needs to use the
 * whole box.  A ticket encodes its device; tickets are waited for with b200_box_wait.  Every box entry that takes a key
 * or an SRS returns B200_ERR_INVALID for one made by another box, even one over the same number of devices. */
typedef struct b200_box b200_box;
typedef struct b200_box_srs b200_box_srs;
typedef struct b200_box_pk b200_box_pk;
int b200_box_create(const int* devices, int n_dev, unsigned workers_per_device, b200_box** out);
void b200_box_destroy(b200_box* box);
int b200_box_devices(const b200_box* box);
/* Device i's pool (b200_pool_* calls work on it directly). */
b200_pool* b200_box_pool(b200_box* box, int i);
int b200_box_srs_load(b200_box* box, const uint8_t* points64, size_t n, int window_bits, int check_on_curve,
                      b200_box_srs** out);
void b200_box_srs_free(b200_box* box, b200_box_srs* srs);
/* b200_plonk_preprocess on every device. */
int b200_box_preprocess(b200_box* box, const b200_box_srs* srs, unsigned log_n, size_t num_inputs,
                        const uint64_t* selectors_evals, const uint64_t* perm, const uint64_t* k, b200_box_pk** out);
int b200_box_pk_verifying_key(const b200_box_pk* pk, uint64_t* selector_comms, uint64_t* sigma_comms);
void b200_box_pk_free(b200_box* box, b200_box_pk* pk);
/* b200_pool_submit_prove on the least-loaded device. */
int b200_box_submit_prove(b200_box* box, const b200_box_pk* pk, const uint64_t* wires, const uint64_t* pub_inputs,
                          size_t num_inputs, const uint64_t* blinders, b200_proof* proof, uint64_t* link_poly,
                          uint64_t* ticket);
/* b200_pool_submit_bundle on the least-loaded device: `pks[i]` is the box key of proofs[i] (the `pk` field of the
 * entries is ignored); a bundle stays on one device. */
int b200_box_submit_bundle(b200_box* box, const b200_box_srs* srs, const b200_box_pk* const* pks,
                           const b200_bundle_proof* proofs, size_t n_proofs, const b200_bundle_link* links,
                           size_t n_links, uint64_t* ticket);
/* b200_plonk_preprocess_wiring on every device: a box key whose proofs can be made from witness vectors. */
int b200_box_preprocess_wiring(b200_box* box, const b200_box_srs* srs, unsigned log_n, size_t num_inputs,
                               const uint64_t* selectors_evals, const unsigned* wire_vars, size_t num_vars,
                               const uint64_t* k, b200_box_pk** out);
/* b200_pool_submit_prove_witness on one device of the box.  A witness in device memory runs on the device that holds it
 * (the least loaded of the box entries with that ordinal); host, pinned and managed witnesses go to the least-loaded
 * device.  B200_ERR_INVALID for a witness on a device outside the box, a key of another box or a key without wiring. */
int b200_box_submit_prove_witness(b200_box* box, const b200_box_pk* pk, const uint64_t* witness, const uint64_t* blinders,
                                  b200_proof* proof, uint64_t* link_poly, uint64_t* pub_inputs_out, uint64_t* ticket);
/* b200_pool_submit_bundle_witness on one device of the box: `pks[i]` is the box key of proofs[i] (the `pk` field of the
 * entries is ignored).  The bundle stays on one device, chosen as for b200_box_submit_prove_witness; a bundle whose
 * device-memory witnesses lie on two different devices is refused with B200_ERR_INVALID. */
int b200_box_submit_bundle_witness(b200_box* box, const b200_box_srs* srs, const b200_box_pk* const* pks,
                                   const b200_bundle_witness* proofs, size_t n_proofs, const b200_bundle_link* links,
                                   size_t n_links, uint64_t* ticket);
int b200_box_wait(b200_box* box, uint64_t ticket);
/* Index (into the `devices` array) of the device a ticket ran on, -1 for a bad ticket. */
int b200_box_ticket_device(const b200_box* box, uint64_t ticket);

/* ---- multi-GPU: one MSM sharded over the GPUs of a box (SURVEY.md §8(e), boundary B1's
 * `b200_init(const int* devs, int n_dev, ...)`) ----------------------------------------------------
 * Rank g of W owns the points [g n / W, (g + 1) n / W) (b200_shard_range) with resident window tables
 * and gets the matching scalar slice; every GPU runs the whole Pippenger on its shard and contributes
 * ONE group element; the exchange is one `ncclAllGather` of the W 128-byte records over NVLink and a
 * W-term addition on every device, in rank order — the affine result is bit-identical to the
 * single-GPU MSM (G1 addition is associative).  NTT and whole proofs do not shard: use one context /
 * one prover pool per device for those.
 * NCCL is bound at run time (libnccl.so.2); the calls fail with B200_ERR_INVALID when it is absent. */
typedef struct b200_multi b200_multi;             /* contexts + NCCL communicator(s) */
typedef struct b200_multi_bases b200_multi_bases; /* point-range shards of one set of bases */
/* [begin, end) of rank `rank` of `world` over n items (sizes differ by at most one).  Host only. */
void b200_shard_range(size_t n, int rank, int world, size_t* begin, size_t* end);
/* One host process drives all `n_dev` devices (world = n_dev; rank i = devices[i]). */
int b200_multi_init(const int* devices, int n_dev, b200_multi** out);
/* One process per GPU (torchrun): rank 0 makes the id, the host hands it to every rank. */
int b200_nccl_unique_id(uint8_t out[128]);
int b200_multi_init_rank(int device, int rank, int world, const uint8_t unique_id[128], b200_multi** out);
void b200_multi_shutdown(b200_multi* m);
/* NCCL_VERSION_CODE of the library bound at run time. */
int b200_nccl_version(int* version);
int b200_multi_world(const b200_multi* m);
/* devices driven by THIS process (n_dev, or 1 in rank mode), their contexts and global ranks */
int b200_multi_local_devices(const b200_multi* m);
b200_ctx* b200_multi_ctx(b200_multi* m, int local);
int b200_multi_rank(const b200_multi* m, int local);
/* Uploads, for each local device, its range of the n points (the full array is passed) and builds the
 * window tables there; cf. b200_bases_load. */
int b200_multi_bases_load(b200_multi* m, const uint8_t* points64, size_t n, int window_bits,
                          int check_on_curve, b200_multi_bases** out);
/* Synthetic known-discrete-log bases (SURVEY.md §8(d)), generated on each device for its range. */
int b200_multi_bases_known_dlog(b200_multi* m, uint64_t seed, size_t n, int window_bits,
                                b200_multi_bases** out);
void b200_multi_bases_free(b200_multi* m, b200_multi_bases* bases);
size_t b200_multi_bases_len(const b200_multi_bases* bases);
int b200_multi_bases_shard(const b200_multi_bases* bases, int local, size_t* begin, size_t* end);
/* b200_bases_plan of local device `local`'s shard (zeros for an empty shard). */
int b200_multi_bases_plan(const b200_multi_bases* bases, int local, int plan[4]);
/* out = sum_{i<n} scalars[i] * bases[i], n = all points.  `scalars`: the FULL host vector (each local
 * device copies its slice).  Collective: in rank mode every rank must call it; all ranks get the result. */
int b200_multi_msm(b200_multi* m, const b200_multi_bases* bases, const uint64_t* scalars, size_t n,
                   int scalars_montgomery, uint64_t out_xy[8], int* out_is_identity);
/* Same, handing over only the SLICES of the local devices: scalars_local[i] = the scalars of local
 * device i's range — host pointers (scalars_on_device = 0; copied inside the call) or device pointers on
 * that device (1).  NULL is allowed for an empty shard. */
int b200_multi_msm_local(b200_multi* m, const b200_multi_bases* bases, const void* const* scalars_local,
                         int scalars_on_device, int scalars_montgomery, uint64_t out_xy[8], int* out_is_identity);

/* ---- device-vector primitives (Fr, Montgomery, device pointers) -------------------------------
 * The share arithmetic of a collaborative prover (`MultiproverPlonkKzgSnark`, traits.rs:1136) on top of
 * b200_ntt_device / b200_msm_device: element-wise operations, batch inversion of opened values, polynomial
 * evaluation and division by a linear factor.  Each call synchronises the context's stream. */
/* out[i] = a[i] (op) b[i], or a[i] (op) b[0] when b_is_scalar; op 0 add, 1 sub, 2 mul. */
int b200_fr_vec_op(b200_ctx* ctx, int op, const void* d_a, const void* d_b, int b_is_scalar, size_t n, void* d_out);
/* data[i] <- 1 / data[i] in place (0 stays 0). */
int b200_fr_batch_inverse_device(b200_ctx* ctx, void* d_data, size_t n);
/* out = p(z) for the len coefficients at d_coeffs. */
int b200_fr_poly_eval_device(b200_ctx* ctx, const void* d_coeffs, size_t len, const uint64_t z[4], uint64_t out[4]);
/* q = p / (X - z), remainder dropped (len - 1 coefficients written to d_q). */
int b200_fr_poly_div_linear_device(b200_ctx* ctx, const void* d_p, size_t len, const uint64_t z[4], void* d_q);

/* ---- witness-side batch hashing (SURVEY.md §8(f) f4) ------------------------------------- */
/* Every field element these four calls read (states, inputs, leaf hashes, sisters, seeds) must be a canonical
 * Montgomery residue, i.e. < r as a 256-bit integer: the kernels' reductions assume it and do not check it. */
/* `batch` independent Poseidon2 sponge hashes of `len` scalars each (inputs: batch x len x 4
 * limbs, Montgomery; out: batch x 4 limbs; host or device pointers).  Each equals the reference's
 * `compute_poseidon_hash(&values)` / `Poseidon2Sponge::new().hash(&values)`
 * (crates/crypto/src/hash/mod.rs:12-18, poseidon2.rs:38-44): t = 3, rate 2, R_F = 8, R_P = 56,
 * alpha = 5, constants of crates/crypto/src/hash/constants.rs. */
int b200_poseidon2_hash_batch(b200_ctx* ctx, const uint64_t* inputs, size_t batch, size_t len,
                              uint64_t* out);
/* `batch` bare permutations of 3-element states, in place (`Poseidon2Sponge::permute`,
 * poseidon2.rs:90-110). */
int b200_poseidon2_permute_batch(b200_ctx* ctx, uint64_t* states, size_t batch);

/* Roots of `batch` Merkle openings of `height` levels: leaf_hashes[i] is hashed up with its sister nodes
 * (sisters[i * height + lvl], bottom-up); is_right[i * height + lvl] != 0 means the running hash is the RIGHT child at
 * that level, i.e. the node is H(sister, cur), else H(cur, sister) — two-to-one Poseidon2 sponge hashes.  The native
 * side of `PoseidonMerkleHashGadget::compute_root` (circuits-core/src/zk_gadgets/primitives/merkle.rs:13-126) /
 * `MerkleOpening::compute_root`, for the batches witness generation walks (state_wrapper.rs:125-247). */
int b200_poseidon2_merkle_root_batch(b200_ctx* ctx, const uint64_t* leaf_hashes, const uint64_t* sisters,
                                     const uint8_t* is_right, size_t batch, unsigned height, uint64_t* roots);
/* `count` consecutive outputs of `batch` Poseidon CSPRNG streams (darkpool-types/src/csprng.rs:30-75: value i of a
 * stream is H(seed, i)): out[s * count + j] = H(seeds[s], first_index[s] + j).  The share / recovery streams behind
 * every `StateWrapper` (stream-cipher pads, recovery identifiers). */
int b200_poseidon2_csprng_batch(b200_ctx* ctx, const uint64_t* seeds, const uint64_t* first_index, size_t batch,
                                size_t count, uint64_t* out);

/* Keccak-256 of the transcript (host; exported so the hash can be pinned by known answers). */
void b200_keccak256(const uint8_t* data, size_t len, uint8_t out[32]);

/* ---- device self-test ------------------------------------------------------------------ */
/* Runs `iters` random Fr and Fq products through the production multiplier (IMAD.WIDE chains)
 * and the word-serial reference multiplier on the device and returns the number of
 * mismatches in *mismatches (0 expected). */
int b200_selftest_field(b200_ctx* ctx, uint64_t seed, size_t iters, uint64_t* mismatches);
/* out[i] = a[i] (op) b[i] on the device; field: 0 = Fr, 1 = Fq; op: 0 mul, 1 add, 2 sub,
 * 3 inverse of a, 4 square of a (the dedicated squarer), 5 a[i] b[i] + a[j] b[j] and
 * 6 a[i] b[i] - a[j] b[j] with j = n - 1 - i (the fused two-product forms of the curve additions).
 * Host buffers, n x 4 limbs (Montgomery).  For parity tests. */
int b200_field_op(b200_ctx* ctx, int field, int op, const uint64_t* a, const uint64_t* b, size_t n,
                  uint64_t* out);

#ifdef __cplusplus
}
#endif
#endif /* B200PROVER_H */
