/* b200compact.h — compact proving keys for libb200prover: the domains up to 2^23 on one 80 GB H100.
 *
 * A default key (b200_plonk_preprocess) keeps the evaluations of its 13 selectors and 5 sigmas on all six quotient
 * cosets, 18 x 6n field elements, and its prover keeps the wires, public input and z there too: about 110 GiB for a key
 * and one proof at n = 2^23.  A compact key keeps coefficients only.  Round 3 then evaluates the key's 18 polynomials and
 * the proof's 7 on one coset at a time, runs the gate and permutation identity there and moves to the next coset, so
 * those tables shrink to n-element buffers.  Every proof, link hint and verifying key is byte for byte what the default
 * key of the same circuit gives.  The price is time: round 3 of a compact key makes about 6 x (18 + 7) size-n
 * transforms per proof where a default key makes 6 x 1, and the wire and public-input transforms that a default key
 * runs on a side stream underneath the round-2 commitment become part of round 3.
 *
 * A job layer over b200prover.h, declared in a header of its own with the same conventions (libb200prover.so):
 *   - b200_plonk_preprocess_compact and b200_plonk_preprocess_wiring_compact take the arguments of
 *     b200_plonk_preprocess and b200_plonk_preprocess_wiring and return a b200_pk that every prover entry point taking
 *     a b200_pk accepts: b200_plonk_prove, b200_plonk_prove_witness, both b200_plonk_prove*_batch forms, the settlement
 *     entry points of b200settlement.h, and the pool's proof, witness, batch, bundle and settlement jobs.  Free it with
 *     b200_pk_free.  The verifying key (b200_pk_verifying_key) is the default key's.
 *   - The key holds the selector and sigma coefficients, the sigma evaluations on H, the domain's points, the four
 *     per-coset point tables (evaluation points, 1 / (n (x - 1)), s_j^i and s_j^-i, 4 x 6n: kept rather than recomputed
 *     per proof) and, from the wiring, the wiring.  Preprocessing transforms in batches of n-element polynomials and
 *     commits the selectors at most five at a time, so that its scratch stays within what a proof uses.
 *   - A context that proves with a default key and a compact key of the same circuit keeps separate captured graphs for
 *     each, as for any two keys.
 *   - Keys of the multi-GPU box (b200_box_preprocess*) are always default keys: compact box keys are not provided.
 */
#ifndef B200COMPACT_H
#define B200COMPACT_H

#include "b200prover.h"

/* entries of b200_plonk_footprint's out[], in bytes:
 *   0 key                 the proving key, with the wiring (a key from a permutation takes 5 n x 4 bytes less)
 *   1 ntt_scratch         the context's NTT scratch: preprocessing's, and a single proof's
 *   2 domain              the domain's twiddles and coset tables
 *   3 srs                 n + 3 SRS powers with one precomputed window table per window (what an idle GPU gets)
 *   4 msm_scratch         the context's MSM scratch: preprocessing's commitments and a single proof's
 *   5 runtime             an allowance, not an allocation of the library's: the CUDA runtime and the library's modules
 *                         (about 0.5 GiB measured on an H100 80GB HBM3), rounded up to 1 GiB
 *   6 workspace           a single proof's workspace (k = 1)
 *   7 ntt_scratch2        a single proof's second NTT scratch (k = 1; 0 for a compact key)
 *   8 batch_workspace     a prove_batch call's own buffers, for a chunk of k proofs (k > 1)
 *   9 batch_ntt_scratch
 *  10 batch_ntt_scratch2
 *  11 batch_msm_scratch */
#define B200_FOOTPRINT_PARTS 12

#ifdef __cplusplus
extern "C" {
#endif

/* b200_plonk_preprocess, making a compact key */
int b200_plonk_preprocess_compact(b200_ctx* ctx, const b200_bases* srs, unsigned log_n, size_t num_inputs,
                                  const uint64_t* selectors_evals, const uint64_t* perm, const uint64_t* k, b200_pk** out);
/* b200_plonk_preprocess_wiring, making a compact key */
int b200_plonk_preprocess_wiring_compact(b200_ctx* ctx, const b200_bases* srs, unsigned log_n, size_t num_inputs,
                                         const uint64_t* selectors_evals, const unsigned* wire_vars, size_t num_vars,
                                         const uint64_t* k, b200_pk** out);
/* 1 for a compact key, 0 for a default key or NULL */
int b200_pk_is_compact(const b200_pk* pk);
/* The device bytes one context needs for one key of domain 2^log_n (default, or compact when `compact` is non-zero)
 * and one prover call of k proofs: b200_plonk_prove for k = 1, a prove_batch chunk of k otherwise, part by part (the
 * entries above; parts a call does not use are 0).  An estimate from the library's allocation rules, for choosing a
 * mode before allocating; it touches no device.  B200_ERR_INVALID for a NULL out, log_n outside [2, 25] or k outside
 * [1, 64]. */
int b200_plonk_footprint(unsigned log_n, size_t k, int compact, uint64_t out[12]);

#ifdef __cplusplus
}
#endif
#endif /* B200COMPACT_H */
