// BN254 G1 (y^2 = x^3 + 3 over Fq) group law for the MSM kernels.
//
// Replaces what the reference reaches through ark-ec 0.4.2 short_weierstrass
// `Affine`/`Projective` for `SystemCurveGroup = G1Projective`
// (/root/reference/crates/constants/src/lib.rs:63-69).  Group elements are canonical once
// normalised to affine, so any correct formula set is bit-identical to arkworks' output.
//
// Accumulators use extended Jacobian "XYZZ" coordinates (x = X/ZZ, y = Y/ZZZ, ZZ^3 = ZZZ^2):
// mixed addition costs 8M+2S and needs no inversion; ZZ == 0 encodes the identity.
// Affine points travel as 64 bytes x||y in Montgomery form — byte-identical to a record of the
// reference's SRS file (srs.rs:172-182) — with (0,0) reserved for the identity.
#pragma once
#include "ff.cuh"

namespace b200 {

struct alignas(16) g1_affine {
    fe x, y;
};
struct alignas(16) g1_xyzz {
    fe x, y, zz, zzz;
};

using Fq = FqCfg;

FF_HD bool g1_affine_is_inf(const g1_affine& p) { return fe_is_zero(p.x) && fe_is_zero(p.y); }
FF_HD bool g1_xyzz_is_inf(const g1_xyzz& p) { return fe_is_zero(p.zz); }

FF_HD g1_xyzz g1_xyzz_inf() {
    g1_xyzz r;
    r.x = fe_zero();
    r.y = fe_zero();
    r.zz = fe_zero();
    r.zzz = fe_zero();
    return r;
}

FF_HD g1_affine g1_affine_neg(const g1_affine& p) {
    g1_affine r;
    r.x = p.x;
    r.y = fe_neg<Fq>(p.y);  // fe_neg(0) = 0 keeps the identity encoding
    return r;
}

FF_HD g1_xyzz g1_xyzz_from_affine(const g1_affine& p) {
    g1_xyzz r;
    if (g1_affine_is_inf(p)) return g1_xyzz_inf();
    r.x = p.x;
    r.y = p.y;
    r.zz = fe_one<Fq>();
    r.zzz = fe_one<Fq>();
    return r;
}

// 2*P for affine P (EFD mdbl-2008-s-1, a = 0)
FF_HD g1_xyzz g1_dbl_affine(const g1_affine& p) {
    if (g1_affine_is_inf(p) || fe_is_zero(p.y)) return g1_xyzz_inf();
    g1_xyzz r;
    fe u = fe_dbl<Fq>(p.y);
    fe v = fe_sqr<Fq>(u);
    fe w = fe_mul<Fq>(u, v);
    fe s = fe_mul<Fq>(p.x, v);
    fe xx = fe_sqr<Fq>(p.x);
    fe m = fe_add<Fq>(fe_dbl<Fq>(xx), xx);
    r.x = fe_sub<Fq>(fe_sqr<Fq>(m), fe_dbl<Fq>(s));
    r.y = fe_mul_sub2<Fq>(m, fe_sub<Fq>(s, r.x), w, p.y);
    r.zz = v;
    r.zzz = w;
    return r;
}

// 2*P (EFD dbl-2008-s-1, a = 0)
FF_HD g1_xyzz g1_dbl(const g1_xyzz& p) {
    if (g1_xyzz_is_inf(p) || fe_is_zero(p.y)) return g1_xyzz_inf();
    g1_xyzz r;
    fe u = fe_dbl<Fq>(p.y);
    fe v = fe_sqr<Fq>(u);
    fe w = fe_mul<Fq>(u, v);
    fe s = fe_mul<Fq>(p.x, v);
    fe xx = fe_sqr<Fq>(p.x);
    fe m = fe_add<Fq>(fe_dbl<Fq>(xx), xx);
    r.x = fe_sub<Fq>(fe_sqr<Fq>(m), fe_dbl<Fq>(s));
    r.y = fe_mul_sub2<Fq>(m, fe_sub<Fq>(s, r.x), w, p.y);
    r.zz = fe_mul<Fq>(v, p.zz);
    r.zzz = fe_mul<Fq>(w, p.zzz);
    return r;
}

// acc + P, P affine (EFD madd-2008-s).  Handles identity operands, P == acc (doubling) and
// P == -acc (identity) exactly, so duplicate bases and cancelling terms stay bit-exact.
FF_HD g1_xyzz g1_add_mixed(const g1_xyzz& a, const g1_affine& p) {
    if (g1_affine_is_inf(p)) return a;
    if (g1_xyzz_is_inf(a)) return g1_xyzz_from_affine(p);
    fe u2 = fe_mul<Fq>(p.x, a.zz);
    fe s2 = fe_mul<Fq>(p.y, a.zzz);
    fe pp_ = fe_sub<Fq>(u2, a.x);
    fe rr = fe_sub<Fq>(s2, a.y);
    if (fe_is_zero(pp_)) {
        if (fe_is_zero(rr)) return g1_dbl_affine(p);
        return g1_xyzz_inf();
    }
    g1_xyzz r;
    fe pp = fe_sqr<Fq>(pp_);
    fe ppp = fe_mul<Fq>(pp_, pp);
    fe q = fe_mul<Fq>(a.x, pp);
    r.x = fe_sub<Fq>(fe_sub<Fq>(fe_sqr<Fq>(rr), ppp), fe_dbl<Fq>(q));
    r.y = fe_mul_sub2<Fq>(rr, fe_sub<Fq>(q, r.x), a.y, ppp);
    r.zz = fe_mul<Fq>(a.zz, pp);
    r.zzz = fe_mul<Fq>(a.zzz, ppp);
    return r;
}

// a + b, both XYZZ (EFD add-2008-s) with the same exact edge-case handling.
FF_HD g1_xyzz g1_add(const g1_xyzz& a, const g1_xyzz& b) {
    if (g1_xyzz_is_inf(b)) return a;
    if (g1_xyzz_is_inf(a)) return b;
    fe u1 = fe_mul<Fq>(a.x, b.zz);
    fe u2 = fe_mul<Fq>(b.x, a.zz);
    fe s1 = fe_mul<Fq>(a.y, b.zzz);
    fe s2 = fe_mul<Fq>(b.y, a.zzz);
    fe pp_ = fe_sub<Fq>(u2, u1);
    fe rr = fe_sub<Fq>(s2, s1);
    if (fe_is_zero(pp_)) {
        if (fe_is_zero(rr)) return g1_dbl(a);
        return g1_xyzz_inf();
    }
    g1_xyzz r;
    fe pp = fe_sqr<Fq>(pp_);
    fe ppp = fe_mul<Fq>(pp_, pp);
    fe q = fe_mul<Fq>(u1, pp);
    r.x = fe_sub<Fq>(fe_sub<Fq>(fe_sqr<Fq>(rr), ppp), fe_dbl<Fq>(q));
    r.y = fe_mul_sub2<Fq>(rr, fe_sub<Fq>(q, r.x), s1, ppp);
    r.zz = fe_mul<Fq>(fe_mul<Fq>(a.zz, b.zz), pp);
    r.zzz = fe_mul<Fq>(fe_mul<Fq>(a.zzz, b.zzz), ppp);
    return r;
}

// XYZZ -> affine with one field inversion:  1/ZZ = ZZ^2 / ZZZ^2,  x = X/ZZ,  y = Y/ZZZ.
FF_HD g1_affine g1_to_affine(const g1_xyzz& p) {
    g1_affine r;
    if (g1_xyzz_is_inf(p)) {
        r.x = fe_zero();
        r.y = fe_zero();
        return r;
    }
    fe i3 = fe_inv<Fq>(p.zzz);  // 1/ZZZ
    // 1/ZZ = ZZ^2 * (1/ZZZ)^2, because ZZ^2/ZZZ^2 = ZZ^2/ZZ^3
    fe izz = fe_mul<Fq>(fe_sqr<Fq>(p.zz), fe_sqr<Fq>(i3));
    r.x = fe_mul<Fq>(p.x, izz);
    r.y = fe_mul<Fq>(p.y, i3);
    return r;
}

// k*P by double-and-add over the low `bits` bits of a canonical scalar (setup-time helper)
FF_HD g1_xyzz g1_mul_bits(const g1_affine& p, const fe& k, int bits) {
    g1_xyzz acc = g1_xyzz_inf();
    for (int i = bits - 1; i >= 0; --i) {
        acc = g1_dbl(acc);
        if ((k.l[i >> 5] >> (i & 31)) & 1u) acc = g1_add_mixed(acc, p);
    }
    return acc;
}

// also false for a coordinate outside [0, q): (x + q, y) would otherwise pass as a second encoding of (x, y)
FF_HD bool g1_affine_on_curve(const g1_affine& p) {
    if (!fe_is_canonical<Fq>(p.x) || !fe_is_canonical<Fq>(p.y)) return false;
    if (g1_affine_is_inf(p)) return true;
    fe lhs = fe_sqr<Fq>(p.y);
    fe rhs = fe_add<Fq>(fe_mul<Fq>(fe_sqr<Fq>(p.x), p.x), fe_from_u32<Fq>(3));
    return fe_eq(lhs, rhs);
}

#if defined(__CUDACC__)
FF_D g1_affine g1_affine_load_ro(const g1_affine* p) {
    g1_affine r;
    r.x = fe_load_ro(&p->x);
    r.y = fe_load_ro(&p->y);
    return r;
}
FF_D void g1_affine_store(g1_affine* p, const g1_affine& v) {
    fe_store(&p->x, v.x);
    fe_store(&p->y, v.y);
}
FF_D g1_xyzz g1_xyzz_load(const g1_xyzz* p) {
    g1_xyzz r;
    r.x = fe_load(&p->x);
    r.y = fe_load(&p->y);
    r.zz = fe_load(&p->zz);
    r.zzz = fe_load(&p->zzz);
    return r;
}
FF_D void g1_xyzz_store(g1_xyzz* p, const g1_xyzz& v) {
    fe_store(&p->x, v.x);
    fe_store(&p->y, v.y);
    fe_store(&p->zz, v.zz);
    fe_store(&p->zzz, v.zzz);
}
#endif

}  // namespace b200
