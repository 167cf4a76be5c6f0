/* TEST INFRASTRUCTURE — CPU restatement (plain C, gcc) of the BN254 arithmetic under the
 * PlonK prover of renegade-fi/renegade.  Only tests/, __graft_entry__.smoke() and bench.py's
 * cpu_baseline / --impl reference legs may load this library; the product path
 * (renegade_b200/csrc) never links or calls it.
 *
 * PARITY STATUS: "parity unpinned" at proof-byte level — the reference's arithmetic lives in
 * un-vendored Rust crates (ark-ff / ark-ec / ark-poly 0.4.2, ark-bn254 0.4.0, mpc-jellyfish
 * @311568a4: /root/reference/Cargo.lock:933,974,1046,1199,5024) and no Rust toolchain exists
 * here, so oracle/_ref cannot be built.  The reference holds no golden vector for MSM/NTT
 * (SURVEY.md §8c).  Pinned against reference-owned data: the SRS file (srs/srs00.. parsed as
 * crates/circuits/circuit-types/src/primitives/srs.rs:63-209; on-curve check :178-179) and
 * the curve/field choice of crates/constants/src/lib.rs:63-89; cross-pinned against the
 * independent big-int restatement oracle/bn254_py.py and the fixtures under tests/golden.
 *
 * Data formats (identical to arkworks' in-memory layout, SURVEY.md §8(a6)):
 *   field element = 4 x uint64 little-endian limbs; "mont" = a*2^256 mod p, "canon" = a.
 *   G1 affine     = x || y (8 x uint64, Montgomery); infinity flagged separately.
 */
#ifndef BN254_ORACLE_H
#define BN254_ORACLE_H
#include <stddef.h>
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

/* --- field arithmetic (ark-ff 0.4.2 fields/models/fp/montgomery_backend.rs) ------------- */
/* which: 0 = Fr (scalar field), 1 = Fq (base field) */
void orc_fp_mul(int which, const uint64_t a[4], const uint64_t b[4], uint64_t out[4]);
void orc_fp_add(int which, const uint64_t a[4], const uint64_t b[4], uint64_t out[4]);
void orc_fp_sub(int which, const uint64_t a[4], const uint64_t b[4], uint64_t out[4]);
void orc_fp_inv(int which, const uint64_t a[4], uint64_t out[4]);
void orc_fp_to_mont(int which, const uint64_t a[4], uint64_t out[4]);
void orc_fp_from_mont(int which, const uint64_t a[4], uint64_t out[4]);
void orc_fp_array_from_mont(int which, const uint64_t* a, size_t n, uint64_t* out);
void orc_fp_array_to_mont(int which, const uint64_t* a, size_t n, uint64_t* out);

/* --- G1 (ark-ec 0.4.2 short_weierstrass) ------------------------------------------------- */
int orc_g1_on_curve(const uint64_t xy_mont[8]);
/* out = a + b (affine, Montgomery); *_inf flags */
void orc_g1_add(const uint64_t a[8], int a_inf, const uint64_t b[8], int b_inf,
                uint64_t out[8], int* out_inf);
/* out = k * P, k canonical 4 limbs */
void orc_g1_mul(const uint64_t p[8], int p_inf, const uint64_t k_canon[4], uint64_t out[8],
                int* out_inf);

/* --- synthetic inputs (SURVEY.md §8(d)) --------------------------------------------------- */
/* element i = 4 consecutive SplitMix64 outputs (4i..4i+3) as LE limbs, reduced mod r */
void orc_splitmix_fr(uint64_t seed, size_t first, size_t n, int montgomery, uint64_t* out);
/* known-dlog bases P_i = a_i * G, a_i = splitmix_fr(seed)[first + i]; out n x 8 limbs (Montgomery) */
void orc_g1_known_dlog_bases(uint64_t seed, size_t first, size_t n, uint64_t* out_xy);

/* sum_i a_i b_i mod r (canonical) over i < n, a_i = splitmix_fr(seed_a)[first_a + i], b_i = splitmix_fr(seed_b)[first_b + i]
 * (OpenMP): the discrete log of an MSM of known-dlog bases with SplitMix scalars */
void orc_fr_dot(uint64_t seed_a, size_t first_a, uint64_t seed_b, size_t first_b, size_t n, uint64_t out_canon[4]);

/* --- MSM: restates ark-ec 0.4.2 VariableBaseMSM::msm_bigint (SURVEY.md App. B) ------------ */
/* scalars canonical (BigInt<4>), bases affine Montgomery; threads across windows (OpenMP,
 * like arkworks' rayon cfg_into_iter over windows). */
void orc_msm(const uint64_t* bases_xy, const uint64_t* scalars_canon, size_t n,
             uint64_t out_xy[8], int* out_inf);
/* definition: sum of double-and-add products (slow; small n only) */
void orc_msm_naive(const uint64_t* bases_xy, const uint64_t* scalars_canon, size_t n,
                   uint64_t out_xy[8], int* out_inf);
int orc_msm_window_bits(size_t n);

/* --- NTT: restates ark-poly 0.4.2 Radix2EvaluationDomain::{fft,ifft,coset_fft,coset_ifft} -- */
/* data: n = 2^log_n Montgomery elements, natural order in and out, in place.
 * inverse: scales by n^-1.  coset: shift g = Fr::GENERATOR = 5. */
void orc_ntt(uint64_t* data, unsigned log_n, int inverse, int coset);
void orc_domain_generator(unsigned log_n, uint64_t out_mont[4]);

/* --- Poseidon2, t = 3 (crates/crypto/src/hash/poseidon2.rs:25-209; poseidon2_oracle.c) ----------------- */
/* full_rc: 24 x 4 limbs, partial_rc: 56 x 4 limbs, both Montgomery; states / inputs / out Montgomery. */
/* `batch` permutations of 3-element states, in place */
void orc_poseidon2_permute_batch(uint64_t* states, size_t batch, const uint64_t* full_rc, const uint64_t* partial_rc);
/* out[i] = sponge hash of inputs[i * len .. (i + 1) * len) (absorb at rate 2, one squeeze) */
void orc_poseidon2_hash_batch(const uint64_t* inputs, size_t batch, size_t len, const uint64_t* full_rc,
                              const uint64_t* partial_rc, uint64_t* out);

int orc_num_threads(void);
void orc_set_num_threads(int n);

#ifdef __cplusplus
}
#endif
#endif
