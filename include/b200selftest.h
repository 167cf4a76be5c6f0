/* b200selftest.h — the device self-test of libb200prover's pairing arithmetic, beside b200_selftest_field
 * (b200prover.h), in a header of its own with the same conventions and error codes (libb200prover.so).
 *
 * b200_pairing_check_many and b200_plonk_verify_each spread each check's Fq12 arithmetic over a group of 16 lanes while
 * the checks fit in one wave of the device, and run each check on one thread past that.  This self-test holds the
 * group arithmetic equal to the one-thread functions, operation by operation. */
#ifndef B200SELFTEST_H
#define B200SELFTEST_H

#include "b200prover.h"

#ifdef __cplusplus
extern "C" {
#endif

/* Runs `iters` seeded Fq12 operands through the 16-lane pairing arithmetic and through the one-thread pairing functions
 * on the device: products, squares, sparse line products, conjugation, both Frobenius maps, inverses, exponentiations
 * by the curve parameter, final exponentiations and a Miller loop over two prepared G2 points (the generator and its
 * negation).  Operands include dense values, values with zero coefficients, 1 and 0.  *mismatches = the number of
 * results that differ in any coefficient (0 expected).  B200_ERR_NO_DEVICE without a CUDA device; B200_ERR_INVALID for
 * a NULL handle or output. */
int b200_selftest_pairing(b200_ctx* ctx, uint64_t seed, size_t iters, uint64_t* mismatches);

#ifdef __cplusplus
}
#endif
#endif /* B200SELFTEST_H */
