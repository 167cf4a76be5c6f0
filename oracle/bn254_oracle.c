/* TEST INFRASTRUCTURE — see bn254_oracle.h for scope, citations and parity status. */
#include "bn254_oracle.h"

#include <stdlib.h>
#include <string.h>
#ifdef _OPENMP
#include <omp.h>
#endif

#include "bn254_internal.h"

void orc_fp_mul(int w, const u64 a[4], const u64 b[4], u64 o[4]) { fp_mul(params(w), o, a, b); }
void orc_fp_add(int w, const u64 a[4], const u64 b[4], u64 o[4]) { fp_add(params(w), o, a, b); }
void orc_fp_sub(int w, const u64 a[4], const u64 b[4], u64 o[4]) { fp_sub(params(w), o, a, b); }
void orc_fp_inv(int w, const u64 a[4], u64 o[4]) { fp_inv(params(w), o, a); }
void orc_fp_to_mont(int w, const u64 a[4], u64 o[4]) { fp_to_mont(params(w), o, a); }
void orc_fp_from_mont(int w, const u64 a[4], u64 o[4]) { fp_from_mont(params(w), o, a); }
void orc_fp_array_from_mont(int w, const u64* a, size_t n, u64* out) {
    const fp_params* P = params(w);
#pragma omp parallel for schedule(static)
    for (size_t i = 0; i < n; ++i) fp_from_mont(P, out + 4 * i, a + 4 * i);
}
void orc_fp_array_to_mont(int w, const u64* a, size_t n, u64* out) {
    const fp_params* P = params(w);
#pragma omp parallel for schedule(static)
    for (size_t i = 0; i < n; ++i) fp_to_mont(P, out + 4 * i, a + 4 * i);
}

int orc_g1_on_curve(const u64 xy[8]) {
    const fp_params* F = &FQ;
    u64 lhs[4], rhs[4], three[4] = {3, 0, 0, 0}, b[4];
    fp_to_mont(F, b, three);
    fp_sqr(F, lhs, xy + 4);
    fp_sqr(F, rhs, xy);
    fp_mul(F, rhs, rhs, xy);
    fp_add(F, rhs, rhs, b);
    return eq4(lhs, rhs);
}

void orc_g1_add(const u64 a[8], int a_inf, const u64 b[8], int b_inf, u64 out[8], int* out_inf) {
    aff A, B, Rr; jac J;
    aff_load(&A, a, a_inf); aff_load(&B, b, b_inf);
    jac_set_inf(&J);
    jac_add_affine(&J, &J, &A);
    jac_add_affine(&J, &J, &B);
    jac_to_affine(&Rr, &J);
    aff_store(&Rr, out, out_inf);
}

static void jac_mul(jac* r, const aff* p, const u64 k[4]) {
    jac acc; jac_set_inf(&acc);
    for (int i = 255; i >= 0; --i) {
        jac_double(&acc, &acc);
        if ((k[i / 64] >> (i % 64)) & 1) jac_add_affine(&acc, &acc, p);
    }
    *r = acc;
}

void orc_g1_mul(const u64 p[8], int p_inf, const u64 k[4], u64 out[8], int* out_inf) {
    aff A, Rr; jac J;
    aff_load(&A, p, p_inf);
    jac_mul(&J, &A, k);
    jac_to_affine(&Rr, &J);
    aff_store(&Rr, out, out_inf);
}

/* batch Jacobian -> affine with one inversion (Montgomery's trick) */
static void jac_batch_to_affine(aff* out, const jac* in, size_t n) {
    const fp_params* F = &FQ;
    u64* pre = (u64*)malloc(n * 32);
    u64 acc[4];
    memcpy(acc, F->r1, 32);
    for (size_t i = 0; i < n; ++i) {
        memcpy(pre + 4 * i, acc, 32);
        if (!jac_is_inf(&in[i])) fp_mul(F, acc, acc, in[i].z);
    }
    u64 inv[4];
    fp_inv(F, inv, acc);
    for (size_t i = n; i-- > 0;) {
        if (jac_is_inf(&in[i])) { memset(&out[i], 0, sizeof(aff)); out[i].inf = 1; continue; }
        u64 zi[4], zi2[4], zi3[4];
        fp_mul(F, zi, inv, pre + 4 * i);
        fp_mul(F, inv, inv, in[i].z);
        fp_sqr(F, zi2, zi);
        fp_mul(F, zi3, zi2, zi);
        fp_mul(F, out[i].x, in[i].x, zi2);
        fp_mul(F, out[i].y, in[i].y, zi3);
        out[i].inf = 0;
    }
    free(pre);
}

/* ------------------------------------------------------------------------------------------
 * Synthetic inputs
 * ---------------------------------------------------------------------------------------- */
static inline u64 splitmix_at(u64 seed, u64 j) { /* j-th output (0-based) of SplitMix64(seed) */
    u64 z = seed + (j + 1) * 0x9E3779B97F4A7C15ULL;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ULL;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBULL;
    return z ^ (z >> 31);
}
static void splitmix_fr_one(u64 seed, u64 i, u64 out_canon[4]) {
    u64 v[4];
    for (int k = 0; k < 4; ++k) v[k] = splitmix_at(seed, 4 * i + k);
    /* 2^256 / r < 6: reduce by repeated subtraction */
    while (ge4(v, FR.p)) sub4(v, v, FR.p);
    memcpy(out_canon, v, 32);
}
void orc_splitmix_fr(u64 seed, size_t first, size_t n, int montgomery, u64* out) {
#pragma omp parallel for schedule(static)
    for (size_t i = 0; i < n; ++i) {
        u64 v[4];
        splitmix_fr_one(seed, first + i, v);
        if (montgomery) fp_to_mont(&FR, out + 4 * i, v);
        else memcpy(out + 4 * i, v, 32);
    }
}

/* sum_i a_i b_i mod r over i < n, a_i = splitmix_fr(seed_a)[first_a + i], b_i = splitmix_fr(seed_b)[first_b + i]: the
 * discrete log of an MSM of n known-dlog bases with SplitMix scalars, without holding either vector.  Montgomery
 * products of canonical operands carry one factor R^-1, which the final to_mont removes. */
void orc_fr_dot(u64 seed_a, size_t first_a, u64 seed_b, size_t first_b, size_t n, u64 out_canon[4]) {
    const size_t chunk = (size_t)1 << 14, n_chunks = (n + chunk - 1) / chunk;
    u64* part = (u64*)calloc(n_chunks ? n_chunks * 4 : 4, sizeof(u64));
#pragma omp parallel for schedule(static)
    for (size_t c = 0; c < n_chunks; ++c) {
        const size_t end = (c + 1) * chunk < n ? (c + 1) * chunk : n;
        u64 acc[4] = {0, 0, 0, 0}, a[4], b[4], t[4];
        for (size_t i = c * chunk; i < end; ++i) {
            splitmix_fr_one(seed_a, first_a + i, a);
            splitmix_fr_one(seed_b, first_b + i, b);
            fp_mul(&FR, t, a, b);
            fp_add(&FR, acc, acc, t);
        }
        memcpy(part + 4 * c, acc, 32);
    }
    u64 sum[4] = {0, 0, 0, 0};
    for (size_t c = 0; c < n_chunks; ++c) fp_add(&FR, sum, sum, part + 4 * c);
    free(part);
    fp_to_mont(&FR, out_canon, sum);
}

void orc_g1_known_dlog_bases(u64 seed, size_t first, size_t n, u64* out_xy) {
    /* table T[b] = 2^b * G (affine) so each base costs popcount(a_i) mixed adds */
    aff* T = (aff*)malloc(256 * sizeof(aff));
    jac* TJ = (jac*)malloc(256 * sizeof(jac));
    jac g; memcpy(g.x, FQ.r1, 32);
    u64 two[4] = {2, 0, 0, 0};
    fp_to_mont(&FQ, g.y, two);
    memcpy(g.z, FQ.r1, 32);
    for (int b = 0; b < 256; ++b) { TJ[b] = g; jac_double(&g, &g); }
    jac_batch_to_affine(T, TJ, 256);
    jac* acc = (jac*)malloc(n * sizeof(jac));
#pragma omp parallel for schedule(static)
    for (size_t i = 0; i < n; ++i) {
        u64 a[4];
        splitmix_fr_one(seed, first + i, a);
        jac J; jac_set_inf(&J);
        for (int b = 0; b < 254; ++b)
            if ((a[b / 64] >> (b % 64)) & 1) jac_add_affine(&J, &J, &T[b]);
        acc[i] = J;
    }
    aff* outa = (aff*)malloc(n * sizeof(aff));
    jac_batch_to_affine(outa, acc, n);
    for (size_t i = 0; i < n; ++i) aff_store(&outa[i], out_xy + 8 * i, NULL);
    free(T); free(TJ); free(acc); free(outa);
}

/* ------------------------------------------------------------------------------------------
 * MSM — ark-ec 0.4.2 msm_bigint restated: c = 3 (n<32) else ceil(log2 n)*69/100 + 2; unsigned
 * c-bit digits over num_bits = 254; each window independently (arkworks: rayon over windows,
 * here: OpenMP); buckets 1..2^c-1; running-sum reduction; Horner with c doublings.
 * ---------------------------------------------------------------------------------------- */
int orc_msm_window_bits(size_t n) {
    if (n < 32) return 3;
    int lg = 0;
    while (((size_t)1 << lg) < n) ++lg; /* ark_std::log2 = ceil */
    return lg * 69 / 100 + 2;
}

void orc_msm(const u64* bases, const u64* scalars, size_t n, u64 out_xy[8], int* out_inf) {
    const int c = orc_msm_window_bits(n);
    const int num_bits = 254;
    const int n_win = (num_bits + c - 1) / c;
    jac* wsum = (jac*)malloc(n_win * sizeof(jac));
#pragma omp parallel for schedule(dynamic, 1)
    for (int w = 0; w < n_win; ++w) {
        const int w_start = w * c;
        const size_t nb = ((size_t)1 << c) - 1;
        jac* buckets = (jac*)malloc(nb * sizeof(jac));
        for (size_t b = 0; b < nb; ++b) jac_set_inf(&buckets[b]);
        for (size_t i = 0; i < n; ++i) {
            const u64* s = scalars + 4 * i;
            if (is_zero4(s)) continue;
            /* digit = (s >> w_start) mod 2^c */
            int limb = w_start / 64, sh = w_start % 64;
            u64 d = s[limb] >> sh;
            if (sh + c > 64 && limb + 1 < 4) d |= s[limb + 1] << (64 - sh);
            d &= ((u64)1 << c) - 1;
            if (d == 0) continue;
            aff P; aff_load(&P, bases + 8 * i, 0);
            jac_add_affine(&buckets[d - 1], &buckets[d - 1], &P);
        }
        jac running, res;
        jac_set_inf(&running); jac_set_inf(&res);
        for (size_t b = nb; b-- > 0;) {
            jac_add(&running, &running, &buckets[b]);
            jac_add(&res, &res, &running);
        }
        wsum[w] = res;
        free(buckets);
    }
    jac total = wsum[n_win - 1];
    for (int w = n_win - 2; w >= 0; --w) {
        for (int k = 0; k < c; ++k) jac_double(&total, &total);
        jac_add(&total, &total, &wsum[w]);
    }
    aff Rr; jac_to_affine(&Rr, &total);
    aff_store(&Rr, out_xy, out_inf);
    free(wsum);
}

void orc_msm_naive(const u64* bases, const u64* scalars, size_t n, u64 out_xy[8], int* out_inf) {
    jac total; jac_set_inf(&total);
    for (size_t i = 0; i < n; ++i) {
        aff P; aff_load(&P, bases + 8 * i, 0);
        jac t; jac_mul(&t, &P, scalars + 4 * i);
        jac_add(&total, &total, &t);
    }
    aff Rr; jac_to_affine(&Rr, &total);
    aff_store(&Rr, out_xy, out_inf);
}

/* ------------------------------------------------------------------------------------------
 * NTT — ark-poly 0.4.2 Radix2EvaluationDomain restated (natural order in/out).
 * ---------------------------------------------------------------------------------------- */
/* TWO_ADIC_ROOT_OF_UNITY = 5^((r-1)/2^28), canonical value (SURVEY.md §8(a5)) */
static const u64 ROOT_2_28_CANON[4] = {0x9bd61b6e725b19f0ULL, 0x402d111e41112ed4ULL,
                                       0x00e0a7eb8ef62abcULL, 0x2a3c09f0a58a7e85ULL};

void orc_domain_generator(unsigned log_n, u64 out[4]) {
    u64 w[4];
    fp_to_mont(&FR, w, ROOT_2_28_CANON);
    for (unsigned i = log_n; i < 28; ++i) fp_sqr(&FR, w, w);
    memcpy(out, w, 32);
}

static size_t bitrev(size_t x, unsigned bits) {
    size_t r = 0;
    for (unsigned i = 0; i < bits; ++i) { r = (r << 1) | (x & 1); x >>= 1; }
    return r;
}

static void distribute_powers(u64* data, size_t n, const u64 g[4]) {
    /* data[i] *= g^i; chunked so it parallelises */
    const size_t chunk = 4096;
#pragma omp parallel for schedule(static)
    for (size_t c0 = 0; c0 < n; c0 += chunk) {
        u64 e[4] = {c0, 0, 0, 0}, t[4];
        fp_pow(&FR, t, g, e);
        size_t end = c0 + chunk < n ? c0 + chunk : n;
        for (size_t i = c0; i < end; ++i) {
            fp_mul(&FR, data + 4 * i, data + 4 * i, t);
            fp_mul(&FR, t, t, g);
        }
    }
}

void orc_ntt(u64* data, unsigned log_n, int inverse, int coset) {
    const size_t n = (size_t)1 << log_n;
    u64 g[4], five[4] = {5, 0, 0, 0};
    fp_to_mont(&FR, g, five);
    if (coset && !inverse) distribute_powers(data, n, g);

    u64 w[4];
    orc_domain_generator(log_n, w);
    if (inverse) fp_inv(&FR, w, w);
    /* twiddle table w^k, k < n/2 */
    size_t half = n / 2 ? n / 2 : 1;
    u64* tw = (u64*)malloc(half * 32);
    {
        const size_t chunk = 2048;
#pragma omp parallel for schedule(static)
        for (size_t c0 = 0; c0 < half; c0 += chunk) {
            u64 e[4] = {c0, 0, 0, 0}, t[4];
            fp_pow(&FR, t, w, e);
            size_t end = c0 + chunk < half ? c0 + chunk : half;
            for (size_t k = c0; k < end; ++k) {
                memcpy(tw + 4 * k, t, 32);
                fp_mul(&FR, t, t, w);
            }
        }
    }
#pragma omp parallel for schedule(static)
    for (size_t i = 0; i < n; ++i) {
        size_t j = bitrev(i, log_n);
        if (i < j) {
            u64 t[4];
            memcpy(t, data + 4 * i, 32);
            memcpy(data + 4 * i, data + 4 * j, 32);
            memcpy(data + 4 * j, t, 32);
        }
    }
    for (size_t m = 1; m < n; m <<= 1) {
        const size_t stride = n / (2 * m);
#pragma omp parallel for schedule(static)
        for (size_t b = 0; b < n / 2; ++b) {
            size_t k = (b / m) * 2 * m, j = b % m;
            u64* u = data + 4 * (k + j);
            u64* v = data + 4 * (k + j + m);
            u64 t[4], s[4];
            fp_mul(&FR, t, v, tw + 4 * (j * stride));
            fp_add(&FR, s, u, t);
            fp_sub(&FR, v, u, t);
            memcpy(u, s, 32);
        }
    }
    free(tw);
    if (inverse) {
        u64 nn[4] = {n, 0, 0, 0}, ninv[4];
        fp_to_mont(&FR, nn, nn);
        fp_inv(&FR, ninv, nn);
#pragma omp parallel for schedule(static)
        for (size_t i = 0; i < n; ++i) fp_mul(&FR, data + 4 * i, data + 4 * i, ninv);
        if (coset) {
            u64 gi[4];
            fp_inv(&FR, gi, g);
            distribute_powers(data, n, gi);
        }
    }
}

void orc_set_num_threads(int n) {
#ifdef _OPENMP
    if (n > 0) omp_set_num_threads(n);
#else
    (void)n;
#endif
}

int orc_num_threads(void) {
#ifdef _OPENMP
    return omp_get_max_threads();
#else
    return 1;
#endif
}
