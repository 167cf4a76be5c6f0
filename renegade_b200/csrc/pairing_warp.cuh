// The BN254 pairing of pairing.cuh with each Fq12 spread over a group of 16 lanes (device only): the latency path of the
// device pairing checks (k_pairing_warp, verify_batch.cu).  pairing.cuh stays the one definition of the arithmetic, the
// Miller loop's lines and the final exponentiation's addition chain; this file restates only how an Fq12 operation is
// shared out over lanes.  b200_selftest_pairing holds every operation here equal to its one-thread counterpart.
//
//   * Layout: lane j < 12 of a group holds coefficient c_j of Fq12 = Fq[w] / (w^12 - 18 w^6 + 82), in registers.  A
//     warp holds two groups (two checks).  Lanes 12 .. 15 shadow lanes 0 .. 3 (same index j, same work) and nothing
//     reads them: 16 is the smallest power-of-two shuffle width that holds 12 coefficients, and two checks per warp
//     keep the groups apart with no cross-group traffic.  Every shuffle names its own group's mask, so the two groups
//     of a warp may diverge (a check with an off-curve point leaves early, an identity G1 point skips its lines).
//   * Product: the convolution t_k = sum_{i + j' = k} a_i b_j' (k = 0 .. 22) is split so that lane j computes t_j
//     (j + 1 products) and t_{j+12} (11 - j products), 12 products on every lane; operands arrive by shuffle.  Then
//     the fixed fold of t_12 .. t_22 (below), with one output per lane.
//   * Sparse line product: only the line's non-zero coefficients (w^0, w^1, w^3, w^7, w^9 for a sloped line; w^0,
//     w^2, w^8 for a vertical one) enter the convolution: 5 or 3 products per lane.
//   * Conjugation and x^(q^2) are lane-local; x^q is a lane-local product and the same fold.
//   * Inversion (once per check, in the easy part of the final exponentiation) by norms instead of the polynomial
//     Euclid of fq12_inv, which would take the one-thread temporaries to a stack: with c = conj(f), g = f c lies in
//     Fq6 (w^2 only), z = g g^(q^2) g^(q^4) lies in Fq2 = Fq + Fq w^6, and
//         1 / f = c (g^(q^2) g^(q^4)) / z,   1 / (z0 + z6 w^6) = (z0 + 18 z6 - z6 w^6) / (z0^2 + 18 z0 z6 + 82 z6^2)
//     (the conjugate of z over s^2 = 18 s - 82, s = w^6): five group products and one Fq inversion.  f = 0 gives 0,
//     as fq12_inv does.
#pragma once
#include "pairing.cuh"

namespace b200 {
namespace pw {

// ---- the fold of the high half ------------------------------------------------------------------------------------
// h_k = t_{12+k}, k = 0 .. 10 (and h_11 = t_23 = 0).  With w^12 = 18 w^6 - 82:
//     k <= 5:  w^(12+k) = 18 w^(6+k) - 82 w^k
//     k >= 6:  w^(12+k) = w^(k-6) w^18, and w^18 = w^6 (18 w^6 - 82) = 18 (18 w^6 - 82) - 82 w^6 = 242 w^6 - 1476,
//              so w^(12+k) = 242 w^k - 1476 w^(k-6)
// so each output takes exactly two high terms, the lane's own h_j and h_(j +- 6):
//     lane j < 6:   c_j = t_j - 82 h_j - 1476 h_(j+6)
//     lane j >= 6:  c_j = t_j + 242 h_j + 18 h_(j-6)
// the sequential fold of fq12_mul (k = 22 down to 12: t_(k-6) += 18 t_k, t_(k-12) -= 82 t_k) as one linear map
// (tests/test_pairing_warp_cpu.py checks the map against that fold).
constexpr int kFoldLowOwn = -82, kFoldLowOther = -1476, kFoldHighOwn = 242, kFoldHighOther = 18;

constexpr int kGroup = 16;  // lanes per Fq12

// Per-lane constants, in shared memory so that a lane indexes them by its coefficient
struct Consts {
    fe one, nine;
    fe fold_own[2], fold_other[2];  // [0] lanes j < 6, [1] lanes j >= 6
    fe gamma[12];                   // x^(q^2): gamma^(j mod 6) for coefficient j
    fe frob_lo[12], frob_hi[12];    // x^q: (w^j)^q = frob_lo[j] w^j + frob_hi[j] w^(j+6)  (frob1[j] with u = w^6 - 9)
};

#if defined(__CUDACC__)
// one thread fills the table; the caller synchronises the block
FF_D void consts_init(Consts* k, const PairingConsts& pc) {
    k->one = fe_one<FqCfg>();
    k->nine = fe_from_u32<FqCfg>(9);
    k->fold_own[0] = fe_neg<FqCfg>(fe_from_u32<FqCfg>(-kFoldLowOwn));
    k->fold_other[0] = fe_neg<FqCfg>(fe_from_u32<FqCfg>(-kFoldLowOther));
    k->fold_own[1] = fe_from_u32<FqCfg>(kFoldHighOwn);
    k->fold_other[1] = fe_from_u32<FqCfg>(kFoldHighOther);
#pragma unroll
    for (int j = 0; j < 12; ++j) {
        k->gamma[j] = pc.gamma_pow[j % 6];
        k->frob_lo[j] = fe_sub<FqCfg>(pc.frob1[j].a, fe_mul<FqCfg>(k->nine, pc.frob1[j].b));
        k->frob_hi[j] = pc.frob1[j].b;
    }
}

struct Lanes {
    unsigned mask;  // the 16 lanes of this thread's group
    int lane;       // 0 .. 15 in the group
    int j;          // the coefficient this lane holds (lanes 12 .. 15: j = lane - 12, shadows)
};
FF_D Lanes lanes() {
    const int t = threadIdx.x & 31;
    Lanes g;
    g.lane = t & 15;
    g.mask = 0xffffu << (t & 16);
    g.j = g.lane < 12 ? g.lane : g.lane - 12;
    return g;
}
FF_D fe shfl(const Lanes& g, const fe& v, int src) {
    fe r;
#pragma unroll
    for (int w = 0; w < 8; ++w) r.l[w] = __shfl_sync(g.mask, v.l[w], src, kGroup);
    return r;
}
FF_D fe sel(bool c, const fe& a, const fe& b) {
    fe r;
#pragma unroll
    for (int w = 0; w < 8; ++w) r.l[w] = c ? a.l[w] : b.l[w];
    return r;
}
// coefficient (j - s) mod 12: the partner of position s in the product that lands on t_j or t_(j+12)
FF_D int partner(const Lanes& g, int s) { return g.j >= s ? g.j - s : g.j - s + 12; }

// c_j from lo = t_j and hi = h_j = t_(j+12)
FF_D fe fold(const Lanes& g, const Consts* k, const fe& lo, const fe& hi) {
    const int hv = g.j >= 6;
    const fe other = shfl(g, hi, hv ? g.j - 6 : g.j + 6);
    return fe_add<FqCfg>(lo, fe_mul_add2<FqCfg>(k->fold_own[hv], hi, k->fold_other[hv], other));
}

// a * b
inline __device__ __noinline__ fe mul(fe a, fe b, const Consts* k) {
    const Lanes g = lanes();
    fe lo = fe_zero(), hi = fe_zero();
#pragma unroll 1
    for (int s = 0; s < 12; ++s) {
        const fe p = fe_mul<FqCfg>(shfl(g, a, s), shfl(g, b, partner(g, s)));
        const bool low = s <= g.j;
        const fe acc = fe_add<FqCfg>(sel(low, lo, hi), p);
        lo = sel(low, acc, lo);
        hi = sel(low, hi, acc);
    }
    return fold(g, k, lo, hi);
}
FF_D fe sqr(const fe& a, const Consts* k) { return mul(a, a, k); }

// x -> x^(q^6): w -> -w
FF_D fe conj(const fe& a) { return (lanes().j & 1) ? fe_neg<FqCfg>(a) : a; }
// x -> x^(q^2)
FF_D fe frob2(const fe& a, const Consts* k) { return fe_mul<FqCfg>(a, k->gamma[lanes().j]); }
// x -> x^q: c_j frob_lo[j] lands on w^j, c_j frob_hi[j] on w^(j+6), then the fold
inline __device__ __noinline__ fe frob1(fe a, const Consts* k) {
    const Lanes g = lanes();
    const bool hv = g.j >= 6;
    const int o = hv ? g.j - 6 : g.j + 6;
    const fe cross = fe_mul<FqCfg>(shfl(g, a, o), k->frob_hi[o]);  // c_o frob_hi[o]: on w^j (j >= 6) or w^(j+12)
    const fe own = fe_mul<FqCfg>(a, k->frob_lo[g.j]);
    return fold(g, k, hv ? fe_add<FqCfg>(own, cross) : own, hv ? fe_zero() : cross);
}

// f * l(P), l one of a prepared point's lines (line_eval_mul): the line's coefficient at w^j is formed on lane j, then
// each non-zero position s is broadcast and multiplied into coefficient j - s (mod 12) of f
template <int N>
FF_D fe sparse_mul(const Lanes& g, const Consts* k, const fe& f, const fe& l, const int (&pos)[N]) {
    fe lo = fe_zero(), hi = fe_zero();
#pragma unroll
    for (int i = 0; i < N; ++i) {
        const int s = pos[i];
        const fe p = fe_mul<FqCfg>(shfl(g, l, s), shfl(g, f, partner(g, s)));
        const bool low = s <= g.j;
        const fe acc = fe_add<FqCfg>(sel(low, lo, hi), p);
        lo = sel(low, acc, lo);
        hi = sel(low, hi, acc);
    }
    return fold(g, k, lo, hi);
}
inline __device__ __noinline__ fe line_mul(fe f, const G2Line* line, fe px, fe py, const Consts* k) {
    const uint32_t kind = line->kind;
    if (kind == kLineNone) return f;
    const Lanes g = lanes();
    const int j = g.j;
    // sloped: -y_P at w^0, (m x_P) at w^1 and w^7, (y_R - m x_R) at w^3 and w^9; vertical: x_P at w^0, -x_R at w^2
    // and w^8 (fq12_put: v = a + b u lands as a - 9 b on w^k and b on w^(k+6)).  Lane j takes (a, b) of its fq2 and
    // forms x * (a - 9 b) or x * b, x = x_P for the slope term and 1 otherwise: one product on every lane.
    const bool sloped = kind == kLineSloped;
    const bool low = sloped ? (j == 1 || j == 3) : j == 2;        // a - 9 b
    const bool high = sloped ? (j == 7 || j == 9) : j == 8;       // b
    const fq2& v = (sloped && (j == 3 || j == 9)) ? line->b : line->a;
    const fe va = fe_load(&v.a), vb = fe_load(&v.b);
    fe y = low ? fe_sub<FqCfg>(va, fe_mul<FqCfg>(k->nine, vb)) : high ? vb : fe_zero();
    if (j == 0) y = sloped ? fe_neg<FqCfg>(py) : px;
    const fe x = sloped && (j == 1 || j == 7) ? px : k->one;
    const fe l = fe_mul<FqCfg>(x, y);
    if (sloped) {
        constexpr int pos[5] = {0, 1, 3, 7, 9};
        return sparse_mul(g, k, f, l, pos);
    }
    constexpr int pos[3] = {0, 2, 8};
    return sparse_mul(g, k, f, l, pos);
}

// 1 / a (see the head of the file); 0 for 0
inline __device__ __noinline__ fe inv(fe a, const Consts* k) {
    const Lanes g = lanes();
    const fe c = conj(a);
    const fe gq = mul(a, c, k);                        // in Fq6
    const fe g2 = frob2(gq, k);
    const fe g24 = mul(g2, frob2(g2, k), k);           // g^(q^2) g^(q^4)
    const fe z = mul(gq, g24, k);                      // in Fq2: z0 + z6 w^6
    const fe z0 = shfl(g, z, 0), z6 = shfl(g, z, 6);
    const fe s = fe_add<FqCfg>(z0, fe_mul<FqCfg>(k->fold_other[1], z6));  // z0 + 18 z6
    const fe n = fe_add<FqCfg>(fe_mul<FqCfg>(z0, s), fe_mul<FqCfg>(fe_from_u32<FqCfg>(82), fe_sqr<FqCfg>(z6)));
    const fe ni = fe_inv<FqCfg>(n);
    const fe zi = g.j == 0 ? fe_mul<FqCfg>(s, ni) : g.j == 6 ? fe_neg<FqCfg>(fe_mul<FqCfg>(z6, ni)) : fe_zero();
    return mul(mul(c, g24, k), zi, k);
}

// t^x, x = 4965661367192848881: fq12_pow's square-and-multiply from the top bit (bit 62)
inline __device__ __noinline__ fe pow_x(fe t, const Consts* k) {
    constexpr uint64_t x = 0x44e992b44a6909f1ULL;
    fe r = t;
#pragma unroll 1
    for (int i = 61; i >= 0; --i) {
        r = sqr(r, k);
        if ((x >> i) & 1) r = mul(r, t, k);
    }
    return r;
}

// final_exponentiation, step for step
inline __device__ __noinline__ fe final_exp(fe f, const Consts* k) {
    fe t = mul(conj(f), inv(f, k), k);
    t = mul(frob2(t, k), t, k);
    const fe y0 = conj(pow_x(t, k));
    const fe y1 = sqr(y0, k);
    const fe y2 = sqr(y1, k);
    fe y3 = mul(y2, y1, k);
    const fe y4 = conj(pow_x(y3, k));
    const fe y5 = sqr(y4, k);
    const fe y6 = pow_x(y5, k);  // conj(y5^(-x))
    y3 = conj(y3);
    const fe y7 = mul(y6, y4, k);
    const fe y8 = mul(y7, y3, k);
    const fe y9 = mul(y8, y1, k);
    const fe y10 = mul(y8, y4, k);
    const fe y11 = mul(y10, t, k);
    const fe y13 = mul(frob1(y9, k), y11, k);
    const fe y14 = mul(frob2(y8, k), y13, k);
    const fe y15 = mul(conj(t), y9, k);
    return mul(frob1(frob2(y15, k), k), y14, k);
}

// miller_loop_prepared over m <= 16 pairs: lane j < m holds G1 point j (x_j, y_j); bit j of `skip` marks an identity
// point, whose pair contributes 1
inline __device__ __noinline__ fe miller(const G2Prepared* q, int m, fe x_j, fe y_j, unsigned skip, const Consts* k) {
    const Lanes g = lanes();
    fe f = g.j == 0 ? k->one : fe_zero();
    int step = 0;
#pragma unroll 1
    for (int i = 63; i >= 0; --i) {
        f = sqr(f, k);
        const bool bit = (kAteLow >> i) & 1;
#pragma unroll 1
        for (int p = 0; p < m; ++p) {
            if ((skip >> p) & 1) continue;
            const fe px = shfl(g, x_j, p), py = shfl(g, y_j, p);
            f = line_mul(f, &q[p].line[step], px, py, k);
            if (bit) f = line_mul(f, &q[p].line[step + 1], px, py, k);
        }
        step += bit ? 2 : 1;
    }
#pragma unroll 1
    for (int p = 0; p < m; ++p) {
        if ((skip >> p) & 1) continue;
        const fe px = shfl(g, x_j, p), py = shfl(g, y_j, p);
        f = line_mul(f, &q[p].line[step], px, py, k);
        f = line_mul(f, &q[p].line[step + 1], px, py, k);
    }
    return f;
}

// [a == 1] over the group's 12 coefficients, on every lane of the group
FF_D bool is_one(const fe& a, const Consts* k) {
    const Lanes g = lanes();
    const bool mine = g.lane >= 12 || fe_eq(a, g.j == 0 ? k->one : fe_zero());
    return (__ballot_sync(g.mask, mine) & g.mask) == g.mask;
}
#endif

}  // namespace pw
}  // namespace b200
