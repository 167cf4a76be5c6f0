// The BN254 optimal-ate pairing, host and device: the ONE definition of the Fq2 / Fq12 arithmetic, the Miller loop's
// line evaluation and the final exponentiation, shared by the host verifiers (verify.cu) and the device pairing checks
// (verify_batch.cu: b200_pairing_check_many, b200_plonk_verify_each).
//
//   * Fq12 = Fq[w] / (w^12 - 18 w^6 + 82) (so Fq2 = Fq[u]/(u^2 + 1) sits inside as u = w^6 - 9), flat coefficients;
//   * G2 on the sextic twist y^2 = x^3 + 3 / (9 + u); Miller loop over 6x + 2 with x = 4965661367192848881 and the two
//     Frobenius line steps; lines evaluated as sparse elements -y_P + (m x_P) w + (y_R - m x_R) w^3;
//   * final exponentiation: the easy part (q^6 - 1)(q^2 + 1), the hard part by the x-addition chain of Fuentes-Castaneda
//     et al. (three exponentiations by x and Frobenius maps).
//
// Every line of the loop depends on Q alone except where it is evaluated at P, so a G2 point is PREPARED once on the host
// (g2_prepare, verify.cu): the kMillerLines lines of its loop, recorded with the branch the step took (identity r,
// vertical line, tangent or chord).  miller_loop_prepared then evaluates them at the G1 points only, on either side.
// The constants of the Frobenius maps (PairingConsts) are computed on the host and passed to the device by value.
#pragma once
#include "ec.cuh"
#include "ff.cuh"

// the large Fq12 routines are called, not inlined, on the device: one copy each instead of one per call site
#if defined(__CUDACC__)
#define PAIR_HD __host__ __device__ __noinline__
#else
#define PAIR_HD
#endif

namespace b200 {

// ---- Fq2 = Fq[u] / (u^2 + 1) ---------------------------------------------------------------------------
struct fq2 {
    fe a, b;  // a + b u
};
FF_HD fq2 fq2_add(const fq2& x, const fq2& y) { return {fe_add<FqCfg>(x.a, y.a), fe_add<FqCfg>(x.b, y.b)}; }
FF_HD fq2 fq2_sub(const fq2& x, const fq2& y) { return {fe_sub<FqCfg>(x.a, y.a), fe_sub<FqCfg>(x.b, y.b)}; }
FF_HD fq2 fq2_neg(const fq2& x) { return {fe_neg<FqCfg>(x.a), fe_neg<FqCfg>(x.b)}; }
FF_HD fq2 fq2_mul(const fq2& x, const fq2& y) {
    const fe aa = fe_mul<FqCfg>(x.a, y.a), bb = fe_mul<FqCfg>(x.b, y.b);
    const fe cross = fe_mul<FqCfg>(fe_add<FqCfg>(x.a, x.b), fe_add<FqCfg>(y.a, y.b));
    return {fe_sub<FqCfg>(aa, bb), fe_sub<FqCfg>(fe_sub<FqCfg>(cross, aa), bb)};
}
FF_HD fq2 fq2_mul_fq(const fq2& x, const fe& s) { return {fe_mul<FqCfg>(x.a, s), fe_mul<FqCfg>(x.b, s)}; }
FF_HD fq2 fq2_sqr(const fq2& x) { return fq2_mul(x, x); }
FF_HD fq2 fq2_inv(const fq2& x) {  // 1 / (a + b u) = (a - b u) / (a^2 + b^2)
    const fe n = fe_inv<FqCfg>(fe_add<FqCfg>(fe_sqr<FqCfg>(x.a), fe_sqr<FqCfg>(x.b)));
    return {fe_mul<FqCfg>(x.a, n), fe_neg<FqCfg>(fe_mul<FqCfg>(x.b, n))};
}
FF_HD bool fq2_is_zero(const fq2& x) { return fe_is_zero(x.a) && fe_is_zero(x.b); }
FF_HD bool fq2_eq(const fq2& x, const fq2& y) { return fe_eq(x.a, y.a) && fe_eq(x.b, y.b); }
inline fq2 fq2_pow(const fq2& a, const uint64_t* e, int limbs) {
    fq2 r = {fe_one<FqCfg>(), fe_zero()};
    for (int i = limbs * 64 - 1; i >= 0; --i) {
        r = fq2_sqr(r);
        if ((e[i >> 6] >> (i & 63)) & 1) r = fq2_mul(r, a);
    }
    return r;
}

struct g2_affine {
    fq2 x, y;
    bool inf;
};

// ---- Fq12 = Fq[w] / (w^12 - 18 w^6 + 82), flat coefficients -----------------------------------------------
struct fq12 {
    fe c[12];
};
FF_HD fq12 fq12_one() {
    fq12 r;
    for (auto& v : r.c) v = fe_zero();
    r.c[0] = fe_one<FqCfg>();
    return r;
}
FF_HD bool fq12_is_one(const fq12& a) {
    if (!fe_eq(a.c[0], fe_one<FqCfg>())) return false;
    for (int i = 1; i < 12; ++i)
        if (!fe_is_zero(a.c[i])) return false;
    return true;
}
inline PAIR_HD fq12 fq12_mul(const fq12& a, const fq12& b) {
    fe t[23];
    for (auto& v : t) v = fe_zero();
    for (int i = 0; i < 12; ++i) {
        if (fe_is_zero(a.c[i])) continue;
        for (int j = 0; j < 12; ++j) t[i + j] = fe_add<FqCfg>(t[i + j], fe_mul<FqCfg>(a.c[i], b.c[j]));
    }
    const fe c18 = fe_from_u32<FqCfg>(18), c82 = fe_from_u32<FqCfg>(82);
    for (int k = 22; k >= 12; --k) {  // w^k = 18 w^(k-6) - 82 w^(k-12)
        if (fe_is_zero(t[k])) continue;
        t[k - 6] = fe_add<FqCfg>(t[k - 6], fe_mul<FqCfg>(c18, t[k]));
        t[k - 12] = fe_sub<FqCfg>(t[k - 12], fe_mul<FqCfg>(c82, t[k]));
    }
    fq12 r;
    for (int i = 0; i < 12; ++i) r.c[i] = t[i];
    return r;
}
// a^2 with the symmetric products taken once: 78 field products instead of 144
inline PAIR_HD fq12 fq12_sqr(const fq12& a) {
    fe t[23];
    for (auto& v : t) v = fe_zero();
    for (int i = 0; i < 12; ++i) {
        if (fe_is_zero(a.c[i])) continue;
        t[2 * i] = fe_add<FqCfg>(t[2 * i], fe_sqr<FqCfg>(a.c[i]));
        const fe twice = fe_dbl<FqCfg>(a.c[i]);
        for (int j = i + 1; j < 12; ++j) t[i + j] = fe_add<FqCfg>(t[i + j], fe_mul<FqCfg>(twice, a.c[j]));
    }
    const fe c18 = fe_from_u32<FqCfg>(18), c82 = fe_from_u32<FqCfg>(82);
    for (int k = 22; k >= 12; --k) {
        if (fe_is_zero(t[k])) continue;
        t[k - 6] = fe_add<FqCfg>(t[k - 6], fe_mul<FqCfg>(c18, t[k]));
        t[k - 12] = fe_sub<FqCfg>(t[k - 12], fe_mul<FqCfg>(c82, t[k]));
    }
    fq12 r;
    for (int i = 0; i < 12; ++i) r.c[i] = t[i];
    return r;
}
// a + b u placed at w^k: u = w^6 - 9
FF_HD void fq12_put(fq12* f, int k, const fq2& v) {
    const fe nine_b = fe_mul<FqCfg>(fe_from_u32<FqCfg>(9), v.b);
    f->c[k] = fe_add<FqCfg>(f->c[k], fe_sub<FqCfg>(v.a, nine_b));
    f->c[k + 6] = fe_add<FqCfg>(f->c[k + 6], v.b);
}
// x -> x^(q^6): w -> -w
FF_HD fq12 fq12_conj(const fq12& a) {
    fq12 r = a;
    for (int i = 1; i < 12; i += 2) r.c[i] = fe_neg<FqCfg>(a.c[i]);
    return r;
}
// inverse by the extended Euclidean algorithm on polynomials over Fq (degree <= 12)
struct poly13 {
    fe c[13];
};
FF_HD int poly_deg(const poly13& p) {
    int d = 12;
    while (d > 0 && fe_is_zero(p.c[d])) --d;
    return d;
}
inline PAIR_HD fq12 fq12_inv(const fq12& a) {
    poly13 lm, hm, low, high;
    for (int i = 0; i < 13; ++i) lm.c[i] = hm.c[i] = low.c[i] = high.c[i] = fe_zero();
    lm.c[0] = fe_one<FqCfg>();
    for (int i = 0; i < 12; ++i) low.c[i] = a.c[i];
    high.c[0] = fe_from_u32<FqCfg>(82);
    high.c[6] = fe_neg<FqCfg>(fe_from_u32<FqCfg>(18));
    high.c[12] = fe_one<FqCfg>();
    while (poly_deg(low) > 0) {
        const int dl = poly_deg(low), dh = poly_deg(high);
        poly13 r, temp = high;
        for (auto& v : r.c) v = fe_zero();
        const fe inv_lead = fe_inv<FqCfg>(low.c[dl]);
        for (int i = dh - dl; i >= 0; --i) {
            r.c[i] = fe_mul<FqCfg>(temp.c[dl + i], inv_lead);
            for (int k = 0; k <= dl; ++k) temp.c[k + i] = fe_sub<FqCfg>(temp.c[k + i], fe_mul<FqCfg>(r.c[i], low.c[k]));
        }
        poly13 nm = hm, nw = high;
        for (int i = 0; i < 13; ++i)
            for (int j = 0; j < 13 - i; ++j) {
                if (fe_is_zero(r.c[j])) continue;
                nm.c[i + j] = fe_sub<FqCfg>(nm.c[i + j], fe_mul<FqCfg>(lm.c[i], r.c[j]));
                nw.c[i + j] = fe_sub<FqCfg>(nw.c[i + j], fe_mul<FqCfg>(low.c[i], r.c[j]));
            }
        hm = lm;
        high = low;
        lm = nm;
        low = nw;
    }
    const fe inv0 = fe_inv<FqCfg>(low.c[0]);
    fq12 out;
    for (int i = 0; i < 12; ++i) out.c[i] = fe_mul<FqCfg>(lm.c[i], inv0);
    return out;
}
inline PAIR_HD fq12 fq12_pow(const fq12& a, const uint64_t* e, int limbs) {
    fq12 r = fq12_one();
    bool started = false;
    for (int i = limbs * 64 - 1; i >= 0; --i) {
        if (started) r = fq12_sqr(r);
        if ((e[i >> 6] >> (i & 63)) & 1) {
            r = started ? fq12_mul(r, a) : a;
            started = true;
        }
    }
    return r;
}

// Frobenius constants: gamma = w^(q^2 - 1) (a sixth root of unity in Fq) scales the coefficients of x^(q^2);
// for the points of the twist, (x, y)^q = (conj(x) * xi^((q-1)/3), conj(y) * xi^((q-1)/2)), xi = 9 + u.
struct PairingConsts {
    fe gamma_pow[6];  // gamma^k
    fq2 twist_frob_x, twist_frob_y;
    fq2 frob1[12];    // (w^k)^q = frob1[k] w^k: powers of xi^((q-1)/6), xi = w^6 = 9 + u
};
const PairingConsts& pairing_consts();  // host, computed once (verify.cu)

// x -> x^(q^2): coefficient of w^k scaled by gamma^(k mod 6)
FF_HD fq12 fq12_frob2(const fq12& a, const PairingConsts& pc) {
    fq12 r;
    for (int k = 0; k < 12; ++k) r.c[k] = fe_mul<FqCfg>(a.c[k], pc.gamma_pow[k % 6]);
    return r;
}
// x -> x^q: the coefficients are in Fq, so x^q = sum_k c_k (w^q)^k = sum_k c_k frob1[k] w^k with frob1[k] in Fq2 = Fq[u],
// u = w^6 - 9; the products land on w^k and w^(k+6) and fold back with w^12 = 18 w^6 - 82
inline PAIR_HD fq12 fq12_frob1(const fq12& a, const PairingConsts& pc) {
    fe t[18];
    for (auto& v : t) v = fe_zero();
    const fe nine = fe_from_u32<FqCfg>(9);
    for (int k = 0; k < 12; ++k) {
        if (fe_is_zero(a.c[k])) continue;
        const fq2& g = pc.frob1[k];
        t[k] = fe_add<FqCfg>(t[k], fe_mul<FqCfg>(a.c[k], fe_sub<FqCfg>(g.a, fe_mul<FqCfg>(nine, g.b))));
        t[k + 6] = fe_add<FqCfg>(t[k + 6], fe_mul<FqCfg>(a.c[k], g.b));
    }
    const fe c18 = fe_from_u32<FqCfg>(18), c82 = fe_from_u32<FqCfg>(82);
    for (int k = 17; k >= 12; --k) {
        t[k - 6] = fe_add<FqCfg>(t[k - 6], fe_mul<FqCfg>(c18, t[k]));
        t[k - 12] = fe_sub<FqCfg>(t[k - 12], fe_mul<FqCfg>(c82, t[k]));
    }
    fq12 r;
    for (int i = 0; i < 12; ++i) r.c[i] = t[i];
    return r;
}

// t^x for the curve parameter x = 4965661367192848881 (63 bits, 28 of them set)
FF_HD fq12 fq12_pow_x(const fq12& t) {
    const uint64_t x[1] = {0x44e992b44a6909f1ULL};
    return fq12_pow(t, x, 1);
}

inline PAIR_HD fq12 final_exponentiation(const fq12& f, const PairingConsts& pc) {
    // easy part: f^((q^6 - 1)(q^2 + 1)); afterwards t is in the cyclotomic subgroup, where the inverse is the conjugate
    fq12 t = fq12_mul(fq12_conj(f), fq12_inv(f));
    t = fq12_mul(fq12_frob2(t, pc), t);
    // hard part (q^4 - q^2 + 1) / r by the addition chain of Fuentes-Castaneda, Knapp and Rodriguez-Henriquez ("Faster
    // hashing to G2", SAC 2011; the schedule ark-ec's bn model uses): three exponentiations by x, Frobenius maps and a
    // dozen products instead of a 762-bit square-and-multiply.  It raises t to c (q^4 - q^2 + 1) / r with a c prime to r
    // (checked on the exponents: tests/test_pairing.py), which is one exactly when the reduced pairing is.
    auto neg_x = [](const fq12& a) { return fq12_conj(fq12_pow_x(a)); };  // a^(-x)
    const fq12 y0 = neg_x(t);
    const fq12 y1 = fq12_sqr(y0);
    const fq12 y2 = fq12_sqr(y1);
    fq12 y3 = fq12_mul(y2, y1);
    const fq12 y4 = neg_x(y3);
    const fq12 y5 = fq12_sqr(y4);
    fq12 y6 = neg_x(y5);
    y3 = fq12_conj(y3);
    y6 = fq12_conj(y6);
    const fq12 y7 = fq12_mul(y6, y4);
    const fq12 y8 = fq12_mul(y7, y3);
    const fq12 y9 = fq12_mul(y8, y1);
    const fq12 y10 = fq12_mul(y8, y4);
    const fq12 y11 = fq12_mul(y10, t);
    const fq12 y13 = fq12_mul(fq12_frob1(y9, pc), y11);
    const fq12 y14 = fq12_mul(fq12_frob2(y8, pc), y13);
    const fq12 y15 = fq12_mul(fq12_conj(t), y9);
    return fq12_mul(fq12_frob1(fq12_frob2(y15, pc), pc), y14);  // q^3 = q o q^2
}

// ---- Miller loop over prepared G2 points ---------------------------------------------------------------------
// 6x + 2, 65 bits: the top bit starts the loop (r = Q), bits 63 .. 0 each take a doubling step and, when set, an
// addition step; then the two Frobenius steps.  64 + 36 + 2 lines in all.
constexpr uint64_t kAteLow = 0x9d797039be763ba8ULL;
constexpr int kMillerLines = 64 + 36 + 2;
enum : uint32_t { kLineNone = 0, kLineVertical = 1, kLineSloped = 2 };
struct G2Line {
    uint32_t kind;  // kLineNone: r or s was the identity, f is left as it is
    fq2 a, b;       // kLineVertical: a = -x_R (the line x_P - x_R w^2); kLineSloped: a = m, b = y_R - m x_R
};
struct G2Prepared {  // the lines of one G2 point's Miller loop, in loop order
    G2Line line[kMillerLines];
};
// host (verify.cu): the schedule of q, recording exactly the branches the affine Miller steps take for it
void g2_prepare(const g2_affine& q, G2Prepared* out);
// host (verify.cu): the same for a 128-byte record x0 || x1 || y0 || y1 (Montgomery); false, and nothing prepared, when
// the point is off the curve or a coordinate is >= q
bool g2_prepare_record(const uint64_t rec[16], G2Prepared* out);
// host (verify.cu): the point of a 128-byte record (all zero: the identity); false when it is off the curve
bool g2_load_record(const uint64_t rec[16], g2_affine* out);

// f <- f * (the line evaluated at P = (px, py)); the sparse operand first: fq12_mul skips its zero coefficients
FF_HD void line_eval_mul(fq12* f, const G2Line& l, const fe& px, const fe& py) {
    if (l.kind == kLineNone) return;
    fq12 line;
    for (auto& v : line.c) v = fe_zero();
    if (l.kind == kLineVertical) {
        line.c[0] = px;
        fq12_put(&line, 2, l.a);
    } else {
        // untwisted slope = m w:  l(P) = m w (x_P - x_R w^2) - (y_P - y_R w^3) = -y_P + (m x_P) w + (y_R - m x_R) w^3
        line.c[0] = fe_neg<FqCfg>(py);
        fq12_put(&line, 1, fq2_mul_fq(l.a, px));
        fq12_put(&line, 3, l.b);
    }
    *f = fq12_mul(line, *f);
}

// Product of the Miller functions of the m pairs (p[j], q[j]) before the final exponentiation: one accumulator, so the
// 64 squarings are shared by all pairs; a pair whose G1 point is the identity contributes 1 and is skipped.
inline PAIR_HD fq12 miller_loop_prepared(const G2Prepared* q, const g1_affine* p, int m) {
    fq12 f = fq12_one();
    int step = 0;
    for (int i = 63; i >= 0; --i) {
        f = fq12_sqr(f);
        const bool bit = (kAteLow >> i) & 1;
        for (int j = 0; j < m; ++j) {
            if (g1_affine_is_inf(p[j])) continue;
            line_eval_mul(&f, q[j].line[step], p[j].x, p[j].y);
            if (bit) line_eval_mul(&f, q[j].line[step + 1], p[j].x, p[j].y);
        }
        step += bit ? 2 : 1;
    }
    for (int j = 0; j < m; ++j) {
        if (g1_affine_is_inf(p[j])) continue;
        line_eval_mul(&f, q[j].line[step], p[j].x, p[j].y);
        line_eval_mul(&f, q[j].line[step + 1], p[j].x, p[j].y);
    }
    return f;
}

}  // namespace b200
