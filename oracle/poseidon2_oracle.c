/* TEST INFRASTRUCTURE — CPU restatement of the Poseidon2 permutation and sponge hash over the BN254 scalar field
 * (crates/crypto/src/hash/poseidon2.rs:25-209: t = 3, rate 2, capacity 1, R_F = 8, R_P = 56, alpha = 5), on the Fr
 * Montgomery arithmetic of bn254_internal.h.  The round constants come from the caller (oracle_c.py reads them from
 * tests/golden/poseidon2.json), never from the product's poseidon2_constants.h, so this checker stays independent of
 * the code under test.  Pinned against the pure-Python restatement bn254_py.poseidon2_permute / poseidon2_hash and the
 * published known answer by tests/test_poseidon2_oracle_cpu.py.  One state per OpenMP iteration, like orc_msm's
 * windows. */
#include "bn254_oracle.h"

#include <omp.h>

#include "bn254_internal.h"

static inline void p2_sbox(u64 x[4]) { /* x^5 */
    u64 x2[4], x4[4];
    fp_sqr(&FR, x2, x);
    fp_sqr(&FR, x4, x2);
    fp_mul(&FR, x, x4, x);
}
/* M_E = circ(2, 1, 1): every element plus the sum of the state */
static inline void p2_external_mds(u64 s[3][4]) {
    u64 sum[4];
    fp_add(&FR, sum, s[0], s[1]);
    fp_add(&FR, sum, sum, s[2]);
    for (int i = 0; i < 3; ++i) fp_add(&FR, s[i], s[i], sum);
}
/* M_I = [[2,1,1],[1,2,1],[1,1,3]]: every element plus the sum, the last one doubled first */
static inline void p2_internal_mds(u64 s[3][4]) {
    u64 sum[4];
    fp_add(&FR, sum, s[0], s[1]);
    fp_add(&FR, sum, sum, s[2]);
    fp_dbl(&FR, s[2], s[2]);
    for (int i = 0; i < 3; ++i) fp_add(&FR, s[i], s[i], sum);
}
static inline void p2_full_round(u64 s[3][4], const u64* full_rc, int r) {
    for (int i = 0; i < 3; ++i) {
        fp_add(&FR, s[i], s[i], full_rc + 4 * (3 * r + i));
        p2_sbox(s[i]);
    }
    p2_external_mds(s);
}
static void p2_permute(u64 s[3][4], const u64* full_rc, const u64* partial_rc) {
    p2_external_mds(s);
    for (int r = 0; r < 4; ++r) p2_full_round(s, full_rc, r);
    for (int r = 0; r < 56; ++r) {
        fp_add(&FR, s[0], s[0], partial_rc + 4 * r);
        p2_sbox(s[0]);
        p2_internal_mds(s);
    }
    for (int r = 4; r < 8; ++r) p2_full_round(s, full_rc, r);
}

void orc_poseidon2_permute_batch(u64* states, size_t batch, const u64* full_rc, const u64* partial_rc) {
#pragma omp parallel for schedule(static)
    for (size_t t = 0; t < batch; ++t) {
        u64 s[3][4];
        memcpy(s, states + 12 * t, sizeof(s));
        p2_permute(s, full_rc, partial_rc);
        memcpy(states + 12 * t, s, sizeof(s));
    }
}

void orc_poseidon2_hash_batch(const u64* inputs, size_t batch, size_t len, const u64* full_rc, const u64* partial_rc,
                              u64* out) {
#pragma omp parallel for schedule(static)
    for (size_t t = 0; t < batch; ++t) {
        u64 s[3][4];
        memset(s, 0, sizeof(s));
        const u64* x = inputs + 4 * len * t;
        int next = 0;
        for (size_t i = 0; i < len; ++i) { /* absorb into state[1..3], permuting when the rate is full */
            if (next == 2) {
                p2_permute(s, full_rc, partial_rc);
                next = 0;
            }
            fp_add(&FR, s[next + 1], s[next + 1], x + 4 * i);
            ++next;
        }
        p2_permute(s, full_rc, partial_rc); /* squeeze: one permutation, state[CAPACITY] out */
        memcpy(out + 4 * t, s[1], 32);
    }
}
