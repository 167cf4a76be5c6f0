// BN254 prime-field arithmetic for sm_90a: 256-bit Montgomery residues as 8 x u32 limbs.
//
// Replaces (on the device) what the reference reaches through ark-ff 0.4.2
// `Fp<MontBackend<FrConfig,4>,4>` / `FqConfig` (types fixed by
// /root/reference/crates/constants/src/lib.rs:63-89; constants SURVEY.md §8(a6)).
// In-memory layout is identical to arkworks': 32 bytes, little-endian limbs, value a*2^256 mod p,
// so host buffers cross the C ABI without conversion.  One element = one 32-byte DRAM sector;
// a thread moves it with two 128-bit accesses.
//
// The multiplier is word-serial Montgomery (CIOS) on the FMA-pipe integer multiplier
// (mad.lo.cc / madc.hi.cc carry chains).  No tensor cores: this is wide-integer modular
// arithmetic, not a contraction.
#pragma once
#include <cstdint>

#if defined(__CUDACC__)
#define FF_HD __host__ __device__ __forceinline__
#define FF_D __device__ __forceinline__
#else
#define FF_HD inline
#define FF_D inline
#endif

namespace b200 {

struct alignas(16) fe {
    uint32_t l[8];
};

// ---------------------------------------------------------------------------------------------
// Field configurations.  Limb getters are constexpr functions (not arrays) so that, after full
// unrolling, every modulus limb becomes an instruction immediate in SASS.
// ---------------------------------------------------------------------------------------------
struct FrCfg {  // scalar field r
    static FF_HD constexpr uint32_t mod(int i) {
        constexpr uint32_t v[8] = {0xf0000001u, 0x43e1f593u, 0x79b97091u, 0x2833e848u,
                                   0x8181585du, 0xb85045b6u, 0xe131a029u, 0x30644e72u};
        return v[i];
    }
    static FF_HD constexpr uint32_t one(int i) {  // R mod r
        constexpr uint32_t v[8] = {0x4ffffffbu, 0xac96341cu, 0x9f60cd29u, 0x36fc7695u,
                                   0x7879462eu, 0x666ea36fu, 0x9a07df2fu, 0x0e0a77c1u};
        return v[i];
    }
    static FF_HD constexpr uint32_t r2(int i) {  // R^2 mod r
        constexpr uint32_t v[8] = {0xae216da7u, 0x1bb8e645u, 0xe35c59e3u, 0x53fe3ab1u,
                                   0x53bb8085u, 0x8c49833du, 0x7f4e44a5u, 0x0216d0b1u};
        return v[i];
    }
    static constexpr uint32_t inv = 0xefffffffu;  // -r^-1 mod 2^32
};

struct FqCfg {  // base field q
    static FF_HD constexpr uint32_t mod(int i) {
        constexpr uint32_t v[8] = {0xd87cfd47u, 0x3c208c16u, 0x6871ca8du, 0x97816a91u,
                                   0x8181585du, 0xb85045b6u, 0xe131a029u, 0x30644e72u};
        return v[i];
    }
    static FF_HD constexpr uint32_t one(int i) {  // R mod q
        constexpr uint32_t v[8] = {0xc58f0d9du, 0xd35d438du, 0xf5c70b3du, 0x0a78eb28u,
                                   0x7879462cu, 0x666ea36fu, 0x9a07df2fu, 0x0e0a77c1u};
        return v[i];
    }
    static FF_HD constexpr uint32_t r2(int i) {  // R^2 mod q
        constexpr uint32_t v[8] = {0x538afa89u, 0xf32cfc5bu, 0xd44501fbu, 0xb5e71911u,
                                   0x0a417ff6u, 0x47ab1effu, 0xcab8351fu, 0x06d89f71u};
        return v[i];
    }
    static constexpr uint32_t inv = 0xe4866389u;  // -q^-1 mod 2^32
};

// ---------------------------------------------------------------------------------------------
// PTX carry-chain primitives (device only)
// ---------------------------------------------------------------------------------------------
#if defined(__CUDA_ARCH__)
namespace ptx {
FF_D uint32_t add_cc(uint32_t a, uint32_t b) {
    uint32_t r;
    asm volatile("add.cc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b));
    return r;
}
FF_D uint32_t addc_cc(uint32_t a, uint32_t b) {
    uint32_t r;
    asm volatile("addc.cc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b));
    return r;
}
FF_D uint32_t addc(uint32_t a, uint32_t b) {
    uint32_t r;
    asm volatile("addc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b));
    return r;
}
FF_D uint32_t sub_cc(uint32_t a, uint32_t b) {
    uint32_t r;
    asm volatile("sub.cc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b));
    return r;
}
FF_D uint32_t subc_cc(uint32_t a, uint32_t b) {
    uint32_t r;
    asm volatile("subc.cc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b));
    return r;
}
FF_D uint32_t subc(uint32_t a, uint32_t b) {
    uint32_t r;
    asm volatile("subc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b));
    return r;
}
FF_D uint32_t mad_lo_cc(uint32_t a, uint32_t b, uint32_t c) {
    uint32_t r;
    asm volatile("mad.lo.cc.u32 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(c));
    return r;
}
FF_D uint32_t madc_lo_cc(uint32_t a, uint32_t b, uint32_t c) {
    uint32_t r;
    asm volatile("madc.lo.cc.u32 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(c));
    return r;
}
FF_D uint32_t mad_hi_cc(uint32_t a, uint32_t b, uint32_t c) {
    uint32_t r;
    asm volatile("mad.hi.cc.u32 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(c));
    return r;
}
FF_D uint32_t madc_hi_cc(uint32_t a, uint32_t b, uint32_t c) {
    uint32_t r;
    asm volatile("madc.hi.cc.u32 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(c));
    return r;
}
FF_D uint32_t madc_hi(uint32_t a, uint32_t b, uint32_t c) {
    uint32_t r;
    asm volatile("madc.hi.u32 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(c));
    return r;
}
// (lo,hi) pair helpers: ptxas fuses each lo/hi pair on the same multiplicands into one
// IMAD.WIDE.U32[.X] with predicate carry-in/out (checked with cuobjdump -sass).
FF_D void wmul(uint32_t& lo, uint32_t& hi, uint32_t a, uint32_t b) {
    asm volatile("mul.lo.u32 %0, %2, %3; mul.hi.u32 %1, %2, %3;" : "=r"(lo), "=r"(hi) : "r"(a), "r"(b));
}
FF_D void wmad_cc(uint32_t& lo, uint32_t& hi, uint32_t a, uint32_t b) {  // starts a carry chain
    asm volatile("mad.lo.cc.u32 %0, %2, %3, %0; madc.hi.cc.u32 %1, %2, %3, %1;"
                 : "+r"(lo), "+r"(hi) : "r"(a), "r"(b));
}
FF_D void wmadc_cc(uint32_t& lo, uint32_t& hi, uint32_t a, uint32_t b) {  // continues a carry chain
    asm volatile("madc.lo.cc.u32 %0, %2, %3, %0; madc.hi.cc.u32 %1, %2, %3, %1;"
                 : "+r"(lo), "+r"(hi) : "r"(a), "r"(b));
}
}  // namespace ptx
#endif

// ---------------------------------------------------------------------------------------------
// Basic helpers (host + device)
// ---------------------------------------------------------------------------------------------
FF_HD bool fe_is_zero(const fe& a) {
    uint32_t x = 0;
#pragma unroll
    for (int i = 0; i < 8; ++i) x |= a.l[i];
    return x == 0;
}
FF_HD bool fe_eq(const fe& a, const fe& b) {
    uint32_t x = 0;
#pragma unroll
    for (int i = 0; i < 8; ++i) x |= a.l[i] ^ b.l[i];
    return x == 0;
}
FF_HD fe fe_zero() {
    fe r;
#pragma unroll
    for (int i = 0; i < 8; ++i) r.l[i] = 0;
    return r;
}
template <class C>
FF_HD fe fe_one() {
    fe r;
#pragma unroll
    for (int i = 0; i < 8; ++i) r.l[i] = C::one(i);
    return r;
}
template <class C>
FF_HD fe fe_r2() {
    fe r;
#pragma unroll
    for (int i = 0; i < 8; ++i) r.l[i] = C::r2(i);
    return r;
}

// ---------------------------------------------------------------------------------------------
// add / sub / neg / dbl : inputs and outputs fully reduced in [0, p)
// ---------------------------------------------------------------------------------------------
template <class C>
FF_HD fe fe_add(const fe& a, const fe& b) {
    fe s, t;
#if defined(__CUDA_ARCH__)
    s.l[0] = ptx::add_cc(a.l[0], b.l[0]);
#pragma unroll
    for (int i = 1; i < 7; ++i) s.l[i] = ptx::addc_cc(a.l[i], b.l[i]);
    s.l[7] = ptx::addc(a.l[7], b.l[7]);  // p < 2^254: no carry out of 256 bits
    t.l[0] = ptx::sub_cc(s.l[0], C::mod(0));
#pragma unroll
    for (int i = 1; i < 8; ++i) t.l[i] = ptx::subc_cc(s.l[i], C::mod(i));
    uint32_t borrow = ptx::subc(0u, 0u);  // 0xffffffff if s < p
#pragma unroll
    for (int i = 0; i < 8; ++i) s.l[i] = borrow ? s.l[i] : t.l[i];
    return s;
#else
    uint64_t c = 0;
    for (int i = 0; i < 8; ++i) {
        c += (uint64_t)a.l[i] + b.l[i];
        s.l[i] = (uint32_t)c;
        c >>= 32;
    }
    int64_t br = 0;
    for (int i = 0; i < 8; ++i) {
        int64_t d = (int64_t)s.l[i] - (int64_t)C::mod(i) + br;
        t.l[i] = (uint32_t)d;
        br = d >> 32;
    }
    return br ? s : t;
#endif
}

template <class C>
FF_HD fe fe_sub(const fe& a, const fe& b) {
    fe d;
#if defined(__CUDA_ARCH__)
    d.l[0] = ptx::sub_cc(a.l[0], b.l[0]);
#pragma unroll
    for (int i = 1; i < 8; ++i) d.l[i] = ptx::subc_cc(a.l[i], b.l[i]);
    uint32_t mask = ptx::subc(0u, 0u);  // all-ones if a < b
    d.l[0] = ptx::add_cc(d.l[0], C::mod(0) & mask);
#pragma unroll
    for (int i = 1; i < 7; ++i) d.l[i] = ptx::addc_cc(d.l[i], C::mod(i) & mask);
    d.l[7] = ptx::addc(d.l[7], C::mod(7) & mask);
    return d;
#else
    int64_t br = 0;
    for (int i = 0; i < 8; ++i) {
        int64_t v = (int64_t)a.l[i] - (int64_t)b.l[i] + br;
        d.l[i] = (uint32_t)v;
        br = v >> 32;
    }
    if (br) {
        uint64_t c = 0;
        for (int i = 0; i < 8; ++i) {
            c += (uint64_t)d.l[i] + C::mod(i);
            d.l[i] = (uint32_t)c;
            c >>= 32;
        }
    }
    return d;
#endif
}

template <class C>
FF_HD fe fe_neg(const fe& a) {
    return fe_sub<C>(fe_zero(), a);
}
template <class C>
FF_HD fe fe_dbl(const fe& a) {
    return fe_add<C>(a, a);
}

// ---------------------------------------------------------------------------------------------
// Montgomery product a*b*2^-256 mod p, reference variant kept for on-device differential tests.
// Word-serial CIOS, 8 rounds; because p < 2^254 the
// running value stays below 2p < 2^255, so the accumulator needs 9 limbs, never 10 ("no-carry"
// property that ark-ff's MontBackend also exploits).
// ---------------------------------------------------------------------------------------------
template <class C>
FF_HD fe fe_mul_chain(const fe& a, const fe& b) {
    uint32_t t[9];
#pragma unroll
    for (int i = 0; i < 9; ++i) t[i] = 0;
#if defined(__CUDA_ARCH__)
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const uint32_t bi = b.l[i];
        // t += a * bi  (low halves, then high halves one limb up)
        t[0] = ptx::mad_lo_cc(a.l[0], bi, t[0]);
#pragma unroll
        for (int j = 1; j < 8; ++j) t[j] = ptx::madc_lo_cc(a.l[j], bi, t[j]);
        t[8] = ptx::addc(0u, 0u);
        t[1] = ptx::mad_hi_cc(a.l[0], bi, t[1]);
#pragma unroll
        for (int j = 1; j < 7; ++j) t[j + 1] = ptx::madc_hi_cc(a.l[j], bi, t[j + 1]);
        t[8] = ptx::madc_hi(a.l[7], bi, t[8]);
        // t = (t + m * p) / 2^32
        const uint32_t m = t[0] * C::inv;
        (void)ptx::mad_lo_cc(m, C::mod(0), t[0]);  // low limb cancels; keeps the carry
#pragma unroll
        for (int j = 1; j < 8; ++j) t[j] = ptx::madc_lo_cc(m, C::mod(j), t[j]);
        t[8] = ptx::addc(t[8], 0u);
        t[0] = ptx::mad_hi_cc(m, C::mod(0), t[1]);
#pragma unroll
        for (int j = 1; j < 7; ++j) t[j] = ptx::madc_hi_cc(m, C::mod(j), t[j + 1]);
        t[7] = ptx::madc_hi(m, C::mod(7), t[8]);
        t[8] = 0;
    }
    fe r, s;
#pragma unroll
    for (int i = 0; i < 8; ++i) r.l[i] = t[i];
    s.l[0] = ptx::sub_cc(r.l[0], C::mod(0));
#pragma unroll
    for (int i = 1; i < 8; ++i) s.l[i] = ptx::subc_cc(r.l[i], C::mod(i));
    uint32_t borrow = ptx::subc(0u, 0u);
#pragma unroll
    for (int i = 0; i < 8; ++i) r.l[i] = borrow ? r.l[i] : s.l[i];
    return r;
#else
    for (int i = 0; i < 8; ++i) {
        uint64_t carry = 0;
        for (int j = 0; j < 8; ++j) {
            uint64_t v = (uint64_t)a.l[j] * b.l[i] + t[j] + carry;
            t[j] = (uint32_t)v;
            carry = v >> 32;
        }
        t[8] = (uint32_t)carry;  // t[8] was 0
        uint32_t m = t[0] * C::inv;
        uint64_t v = (uint64_t)m * C::mod(0) + t[0];
        carry = v >> 32;
        for (int j = 1; j < 8; ++j) {
            v = (uint64_t)m * C::mod(j) + t[j] + carry;
            t[j - 1] = (uint32_t)v;
            carry = v >> 32;
        }
        t[7] = t[8] + (uint32_t)carry;
        t[8] = 0;
    }
    fe r, s;
    for (int i = 0; i < 8; ++i) r.l[i] = t[i];
    int64_t br = 0;
    for (int i = 0; i < 8; ++i) {
        int64_t d = (int64_t)r.l[i] - (int64_t)C::mod(i) + br;
        s.l[i] = (uint32_t)d;
        br = d >> 32;
    }
    return br ? r : s;
#endif
}

// ---------------------------------------------------------------------------------------------
// Montgomery product, production variant: the same word-serial reduction, but every 32x32->64
// product is accumulated with ONE IMAD.WIDE.U32.X.  The running value T is split into an
// "even" array E (aligned at 2^0) and an "odd" array O (aligned at 2^32): products a_j*s with
// even j land 64-bit-aligned in E, odd j in O, so each carry chain is 4 wide multiply-adds.
// After a round T/2^32 = O + E[1] + 2^32*E[2..8]: O becomes the next round's even array,
// E[2..8] its odd array, and the single limb E[1] is folded in with one add.cc whose carry
// (weight 2^32) enters the odd chain.  Bounds: T < 2p before a round, < 2^288 inside one, so
// O never carries out of 8 limbs and E needs 9.   ~128 IMAD.WIDE + ~50 other instructions.
// ---------------------------------------------------------------------------------------------
template <class C>
FF_HD fe fe_mul(const fe& a, const fe& b) {
#if defined(__CUDA_ARCH__)
    uint32_t E[9], O[8];
    {
        const uint32_t s = b.l[0];
        ptx::wmul(O[0], O[1], a.l[1], s);
        ptx::wmul(O[2], O[3], a.l[3], s);
        ptx::wmul(O[4], O[5], a.l[5], s);
        ptx::wmul(O[6], O[7], a.l[7], s);
        ptx::wmul(E[0], E[1], a.l[0], s);
        ptx::wmul(E[2], E[3], a.l[2], s);
        ptx::wmul(E[4], E[5], a.l[4], s);
        ptx::wmul(E[6], E[7], a.l[6], s);
        const uint32_t m = E[0] * C::inv;
        ptx::wmad_cc(O[0], O[1], C::mod(1), m);
        ptx::wmadc_cc(O[2], O[3], C::mod(3), m);
        ptx::wmadc_cc(O[4], O[5], C::mod(5), m);
        ptx::wmadc_cc(O[6], O[7], C::mod(7), m);
        ptx::wmad_cc(E[0], E[1], C::mod(0), m);
        ptx::wmadc_cc(E[2], E[3], C::mod(2), m);
        ptx::wmadc_cc(E[4], E[5], C::mod(4), m);
        ptx::wmadc_cc(E[6], E[7], C::mod(6), m);
        E[8] = ptx::addc(0u, 0u);
    }
#pragma unroll
    for (int i = 1; i < 8; ++i) {
        // T/2^32: even' = O (+ E[1] at limb 0), odd' = E[2..8]
        uint32_t nE[9], nO[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) nE[k] = O[k];
#pragma unroll
        for (int k = 0; k < 7; ++k) nO[k] = E[k + 2];
        nO[7] = 0;
        const uint32_t s = b.l[i];
        nE[0] = ptx::add_cc(nE[0], E[1]);  // carry has weight 2^32 -> odd chain
        ptx::wmadc_cc(nO[0], nO[1], a.l[1], s);
        ptx::wmadc_cc(nO[2], nO[3], a.l[3], s);
        ptx::wmadc_cc(nO[4], nO[5], a.l[5], s);
        ptx::wmadc_cc(nO[6], nO[7], a.l[7], s);
        ptx::wmad_cc(nE[0], nE[1], a.l[0], s);
        ptx::wmadc_cc(nE[2], nE[3], a.l[2], s);
        ptx::wmadc_cc(nE[4], nE[5], a.l[4], s);
        ptx::wmadc_cc(nE[6], nE[7], a.l[6], s);
        nE[8] = ptx::addc(0u, 0u);
        const uint32_t m = nE[0] * C::inv;
        ptx::wmad_cc(nO[0], nO[1], C::mod(1), m);
        ptx::wmadc_cc(nO[2], nO[3], C::mod(3), m);
        ptx::wmadc_cc(nO[4], nO[5], C::mod(5), m);
        ptx::wmadc_cc(nO[6], nO[7], C::mod(7), m);
        ptx::wmad_cc(nE[0], nE[1], C::mod(0), m);
        ptx::wmadc_cc(nE[2], nE[3], C::mod(2), m);
        ptx::wmadc_cc(nE[4], nE[5], C::mod(4), m);
        ptx::wmadc_cc(nE[6], nE[7], C::mod(6), m);
        nE[8] = ptx::addc(nE[8], 0u);
#pragma unroll
        for (int k = 0; k < 9; ++k) E[k] = nE[k];
#pragma unroll
        for (int k = 0; k < 8; ++k) O[k] = nO[k];
    }
    // result = O + E[1..8]  (< 2p), then one conditional subtraction
    fe r, t;
    r.l[0] = ptx::add_cc(O[0], E[1]);
#pragma unroll
    for (int k = 1; k < 7; ++k) r.l[k] = ptx::addc_cc(O[k], E[k + 1]);
    r.l[7] = ptx::addc(O[7], E[8]);
    t.l[0] = ptx::sub_cc(r.l[0], C::mod(0));
#pragma unroll
    for (int k = 1; k < 8; ++k) t.l[k] = ptx::subc_cc(r.l[k], C::mod(k));
    const uint32_t borrow = ptx::subc(0u, 0u);
#pragma unroll
    for (int k = 0; k < 8; ++k) r.l[k] = borrow ? r.l[k] : t.l[k];
    return r;
#else
    // host path (transcript, affine normalisation, linearisation scalars): 4 x 64-bit CIOS
    uint64_t x[4], y[4], p[4], t[6] = {0, 0, 0, 0, 0, 0};
    for (int i = 0; i < 4; ++i) {
        x[i] = (uint64_t)a.l[2 * i] | ((uint64_t)a.l[2 * i + 1] << 32);
        y[i] = (uint64_t)b.l[2 * i] | ((uint64_t)b.l[2 * i + 1] << 32);
        p[i] = (uint64_t)C::mod(2 * i) | ((uint64_t)C::mod(2 * i + 1) << 32);
    }
    // -p^-1 mod 2^64 from the 32-bit constant by one Newton step
    const uint64_t pinv32 = (uint64_t)(0u - C::inv);          // p^-1 mod 2^32
    const uint64_t pinv64 = pinv32 * (2 - p[0] * pinv32);      // p^-1 mod 2^64
    const uint64_t ninv = 0 - pinv64;
    typedef unsigned __int128 u128;
    for (int i = 0; i < 4; ++i) {
        uint64_t carry = 0;
        for (int j = 0; j < 4; ++j) {
            u128 v = (u128)x[j] * y[i] + t[j] + carry;
            t[j] = (uint64_t)v;
            carry = (uint64_t)(v >> 64);
        }
        u128 v = (u128)t[4] + carry;
        t[4] = (uint64_t)v;
        t[5] = (uint64_t)(v >> 64);
        const uint64_t m = t[0] * ninv;
        v = (u128)m * p[0] + t[0];
        carry = (uint64_t)(v >> 64);
        for (int j = 1; j < 4; ++j) {
            v = (u128)m * p[j] + t[j] + carry;
            t[j - 1] = (uint64_t)v;
            carry = (uint64_t)(v >> 64);
        }
        v = (u128)t[4] + carry;
        t[3] = (uint64_t)v;
        t[4] = t[5] + (uint64_t)(v >> 64);
    }
    bool ge = t[4] != 0;
    if (!ge) {
        ge = true;
        for (int i = 3; i >= 0; --i)
            if (t[i] != p[i]) { ge = t[i] > p[i]; break; }
    }
    if (ge) {
        uint64_t borrow = 0;
        for (int i = 0; i < 4; ++i) {
            u128 d = (u128)t[i] - p[i] - borrow;
            t[i] = (uint64_t)d;
            borrow = (uint64_t)(d >> 64) & 1;
        }
    }
    fe r;
    for (int i = 0; i < 4; ++i) {
        r.l[2 * i] = (uint32_t)t[i];
        r.l[2 * i + 1] = (uint32_t)(t[i] >> 32);
    }
    return r;
#endif
}

// ---------------------------------------------------------------------------------------------
// a*b + c*d (Montgomery) with ONE reduction: each round accumulates both partial products before
// the single m*p step, so the pair costs 192 instead of 256 wide multiply-adds.  Bounds: the
// running value stays below a + c + p < 3p < 2^256, inside a round below 2^288 (E needs 9 limbs,
// O never carries out of 8) — checked with exact carry semantics in Python before the PTX was
// written; the device result is cross-checked against two separate products in
// b200_selftest_field.  Used for Y3 = R (Q - X3) - Y1 PPP of the curve additions.
// ---------------------------------------------------------------------------------------------
template <class C>
FF_HD fe fe_mul_add2(const fe& a, const fe& b, const fe& c, const fe& d) {
#if defined(__CUDA_ARCH__)
    uint32_t E[9], O[8];
    {
        const uint32_t s = b.l[0], t = d.l[0];
        ptx::wmul(O[0], O[1], a.l[1], s);
        ptx::wmul(O[2], O[3], a.l[3], s);
        ptx::wmul(O[4], O[5], a.l[5], s);
        ptx::wmul(O[6], O[7], a.l[7], s);
        ptx::wmul(E[0], E[1], a.l[0], s);
        ptx::wmul(E[2], E[3], a.l[2], s);
        ptx::wmul(E[4], E[5], a.l[4], s);
        ptx::wmul(E[6], E[7], a.l[6], s);
        ptx::wmad_cc(O[0], O[1], c.l[1], t);
        ptx::wmadc_cc(O[2], O[3], c.l[3], t);
        ptx::wmadc_cc(O[4], O[5], c.l[5], t);
        ptx::wmadc_cc(O[6], O[7], c.l[7], t);
        ptx::wmad_cc(E[0], E[1], c.l[0], t);
        ptx::wmadc_cc(E[2], E[3], c.l[2], t);
        ptx::wmadc_cc(E[4], E[5], c.l[4], t);
        ptx::wmadc_cc(E[6], E[7], c.l[6], t);
        E[8] = ptx::addc(0u, 0u);
        const uint32_t m = E[0] * C::inv;
        ptx::wmad_cc(O[0], O[1], C::mod(1), m);
        ptx::wmadc_cc(O[2], O[3], C::mod(3), m);
        ptx::wmadc_cc(O[4], O[5], C::mod(5), m);
        ptx::wmadc_cc(O[6], O[7], C::mod(7), m);
        ptx::wmad_cc(E[0], E[1], C::mod(0), m);
        ptx::wmadc_cc(E[2], E[3], C::mod(2), m);
        ptx::wmadc_cc(E[4], E[5], C::mod(4), m);
        ptx::wmadc_cc(E[6], E[7], C::mod(6), m);
        E[8] = ptx::addc(E[8], 0u);
    }
#pragma unroll
    for (int i = 1; i < 8; ++i) {
        uint32_t nE[9], nO[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) nE[k] = O[k];
#pragma unroll
        for (int k = 0; k < 7; ++k) nO[k] = E[k + 2];
        nO[7] = 0;
        const uint32_t s = b.l[i], t = d.l[i];
        nE[0] = ptx::add_cc(nE[0], E[1]);  // carry has weight 2^32 -> first odd chain
        ptx::wmadc_cc(nO[0], nO[1], a.l[1], s);
        ptx::wmadc_cc(nO[2], nO[3], a.l[3], s);
        ptx::wmadc_cc(nO[4], nO[5], a.l[5], s);
        ptx::wmadc_cc(nO[6], nO[7], a.l[7], s);
        ptx::wmad_cc(nE[0], nE[1], a.l[0], s);
        ptx::wmadc_cc(nE[2], nE[3], a.l[2], s);
        ptx::wmadc_cc(nE[4], nE[5], a.l[4], s);
        ptx::wmadc_cc(nE[6], nE[7], a.l[6], s);
        nE[8] = ptx::addc(0u, 0u);
        ptx::wmad_cc(nO[0], nO[1], c.l[1], t);
        ptx::wmadc_cc(nO[2], nO[3], c.l[3], t);
        ptx::wmadc_cc(nO[4], nO[5], c.l[5], t);
        ptx::wmadc_cc(nO[6], nO[7], c.l[7], t);
        ptx::wmad_cc(nE[0], nE[1], c.l[0], t);
        ptx::wmadc_cc(nE[2], nE[3], c.l[2], t);
        ptx::wmadc_cc(nE[4], nE[5], c.l[4], t);
        ptx::wmadc_cc(nE[6], nE[7], c.l[6], t);
        nE[8] = ptx::addc(nE[8], 0u);
        const uint32_t m = nE[0] * C::inv;
        ptx::wmad_cc(nO[0], nO[1], C::mod(1), m);
        ptx::wmadc_cc(nO[2], nO[3], C::mod(3), m);
        ptx::wmadc_cc(nO[4], nO[5], C::mod(5), m);
        ptx::wmadc_cc(nO[6], nO[7], C::mod(7), m);
        ptx::wmad_cc(nE[0], nE[1], C::mod(0), m);
        ptx::wmadc_cc(nE[2], nE[3], C::mod(2), m);
        ptx::wmadc_cc(nE[4], nE[5], C::mod(4), m);
        ptx::wmadc_cc(nE[6], nE[7], C::mod(6), m);
        nE[8] = ptx::addc(nE[8], 0u);
#pragma unroll
        for (int k = 0; k < 9; ++k) E[k] = nE[k];
#pragma unroll
        for (int k = 0; k < 8; ++k) O[k] = nO[k];
    }
    fe r, t;
    r.l[0] = ptx::add_cc(O[0], E[1]);
#pragma unroll
    for (int k = 1; k < 7; ++k) r.l[k] = ptx::addc_cc(O[k], E[k + 1]);
    r.l[7] = ptx::addc(O[7], E[8]);
    // result < 3p: two conditional subtractions
#pragma unroll
    for (int pass = 0; pass < 2; ++pass) {
        t.l[0] = ptx::sub_cc(r.l[0], C::mod(0));
#pragma unroll
        for (int k = 1; k < 8; ++k) t.l[k] = ptx::subc_cc(r.l[k], C::mod(k));
        const uint32_t borrow = ptx::subc(0u, 0u);
#pragma unroll
        for (int k = 0; k < 8; ++k) r.l[k] = borrow ? r.l[k] : t.l[k];
    }
    return r;
#else
    return fe_add<C>(fe_mul<C>(a, b), fe_mul<C>(c, d));
#endif
}
// a*b - c*d
template <class C>
FF_HD fe fe_mul_sub2(const fe& a, const fe& b, const fe& c, const fe& d) {
    return fe_mul_add2<C>(a, b, c, fe_sub<C>(fe_zero(), d));
}

// ---------------------------------------------------------------------------------------------
// Montgomery square.  Same even/odd word-serial scheme as fe_mul, but round i only multiplies
// a_i by the limbs it has not met yet: a^2 = sum_i a_i * (a_i X^i + 2 * sum_{j>i} a_j X^j), and
// 2 * (a >> 32(i+1)) is read off d = 2a (fits 8 limbs: a < 2^254) with the bit that crossed the
// limb boundary masked.  36 + 64 = 100 wide multiply-adds instead of 128.  The running value stays
// below 2a + p < 3p < 2^256 and the result below 2p (validated in Python with exact carries;
// cross-checked against fe_mul(a, a) on the device by b200_selftest_field).
// ---------------------------------------------------------------------------------------------
#if defined(__CUDA_ARCH__)
template <class C, int I>
FF_D void fe_sqr_round(uint32_t (&E)[9], uint32_t (&O)[8], const fe& a, const fe& d) {
    // operand limbs of this round: v_I = a_I, v_{I+1} = d_{I+1} & ~1, v_j = d_j (j >= I+2)
    auto v = [&](int j) -> uint32_t {
        return j == I ? a.l[j] : (j == I + 1 ? (d.l[j] & 0xfffffffeu) : d.l[j]);
    };
    const uint32_t s = a.l[I];
    uint32_t nE[9], nO[8];
    if constexpr (I == 0) {
        ptx::wmul(nO[0], nO[1], v(1), s);
        ptx::wmul(nO[2], nO[3], v(3), s);
        ptx::wmul(nO[4], nO[5], v(5), s);
        ptx::wmul(nO[6], nO[7], v(7), s);
        ptx::wmul(nE[0], nE[1], v(0), s);
        ptx::wmul(nE[2], nE[3], v(2), s);
        ptx::wmul(nE[4], nE[5], v(4), s);
        ptx::wmul(nE[6], nE[7], v(6), s);
        nE[8] = 0;
    } else {
#pragma unroll
        for (int k = 0; k < 8; ++k) nE[k] = O[k];
#pragma unroll
        for (int k = 0; k < 7; ++k) nO[k] = E[k + 2];
        nO[7] = 0;
        nE[8] = 0;
        constexpr int j0 = (I & 1) ? I : I + 1;   // first odd limb index >= I
        constexpr int j0e = (I & 1) ? I + 1 : I;  // first even limb index >= I
        nE[0] = ptx::add_cc(nE[0], E[1]);  // carry (weight 2^32) runs up the odd array
#pragma unroll
        for (int k = 0; k < j0 - 1; ++k) nO[k] = ptx::addc_cc(nO[k], 0u);
        if constexpr (j0 <= 1) ptx::wmadc_cc(nO[0], nO[1], v(1), s);
        if constexpr (j0 <= 3) ptx::wmadc_cc(nO[2], nO[3], v(3), s);
        if constexpr (j0 <= 5) ptx::wmadc_cc(nO[4], nO[5], v(5), s);
        ptx::wmadc_cc(nO[6], nO[7], v(7), s);
        if constexpr (j0e <= 6) {
            // the first product of the even chain starts a fresh carry chain
            if constexpr (j0e == 0) ptx::wmad_cc(nE[0], nE[1], v(0), s);
            if constexpr (j0e == 2) ptx::wmad_cc(nE[2], nE[3], v(2), s);
            if constexpr (j0e < 2) ptx::wmadc_cc(nE[2], nE[3], v(2), s);
            if constexpr (j0e == 4) ptx::wmad_cc(nE[4], nE[5], v(4), s);
            if constexpr (j0e < 4) ptx::wmadc_cc(nE[4], nE[5], v(4), s);
            if constexpr (j0e == 6) ptx::wmad_cc(nE[6], nE[7], v(6), s);
            if constexpr (j0e < 6) ptx::wmadc_cc(nE[6], nE[7], v(6), s);
            nE[8] = ptx::addc(0u, 0u);
        }
    }
    const uint32_t m = nE[0] * C::inv;
    ptx::wmad_cc(nO[0], nO[1], C::mod(1), m);
    ptx::wmadc_cc(nO[2], nO[3], C::mod(3), m);
    ptx::wmadc_cc(nO[4], nO[5], C::mod(5), m);
    ptx::wmadc_cc(nO[6], nO[7], C::mod(7), m);
    ptx::wmad_cc(nE[0], nE[1], C::mod(0), m);
    ptx::wmadc_cc(nE[2], nE[3], C::mod(2), m);
    ptx::wmadc_cc(nE[4], nE[5], C::mod(4), m);
    ptx::wmadc_cc(nE[6], nE[7], C::mod(6), m);
    nE[8] = ptx::addc(nE[8], 0u);
#pragma unroll
    for (int k = 0; k < 9; ++k) E[k] = nE[k];
#pragma unroll
    for (int k = 0; k < 8; ++k) O[k] = nO[k];
}
#endif

template <class C>
FF_HD fe fe_sqr(const fe& a) {
#if defined(__CUDA_ARCH__)
    fe d;  // 2a as a plain 256-bit integer (no reduction: a < 2^254)
#pragma unroll
    for (int k = 7; k >= 1; --k) d.l[k] = (a.l[k] << 1) | (a.l[k - 1] >> 31);
    d.l[0] = a.l[0] << 1;
    uint32_t E[9], O[8];
    fe_sqr_round<C, 0>(E, O, a, d);
    fe_sqr_round<C, 1>(E, O, a, d);
    fe_sqr_round<C, 2>(E, O, a, d);
    fe_sqr_round<C, 3>(E, O, a, d);
    fe_sqr_round<C, 4>(E, O, a, d);
    fe_sqr_round<C, 5>(E, O, a, d);
    fe_sqr_round<C, 6>(E, O, a, d);
    fe_sqr_round<C, 7>(E, O, a, d);
    fe r, t;
    r.l[0] = ptx::add_cc(O[0], E[1]);
#pragma unroll
    for (int k = 1; k < 7; ++k) r.l[k] = ptx::addc_cc(O[k], E[k + 1]);
    r.l[7] = ptx::addc(O[7], E[8]);
    t.l[0] = ptx::sub_cc(r.l[0], C::mod(0));
#pragma unroll
    for (int k = 1; k < 8; ++k) t.l[k] = ptx::subc_cc(r.l[k], C::mod(k));
    const uint32_t borrow = ptx::subc(0u, 0u);
#pragma unroll
    for (int k = 0; k < 8; ++k) r.l[k] = borrow ? r.l[k] : t.l[k];
    return r;
#else
    return fe_mul<C>(a, a);
#endif
}

template <class C>
FF_HD fe fe_to_mont(const fe& a) {
    return fe_mul<C>(a, fe_r2<C>());
}
template <class C>
FF_HD fe fe_from_mont(const fe& a) {
    fe one = fe_zero();
    one.l[0] = 1;
    return fe_mul<C>(a, one);
}

// a^e for a 256-bit exponent given as 8 limbs (square-and-multiply, MSB first)
template <class C>
FF_HD fe fe_pow(const fe& a, const fe& e) {
    fe acc = fe_one<C>();
    for (int i = 255; i >= 0; --i) {
        acc = fe_sqr<C>(acc);
        if ((e.l[i >> 5] >> (i & 31)) & 1u) acc = fe_mul<C>(acc, a);
    }
    return acc;
}

// Fermat inverse a^(p-2); inv(0) = 0.  Kept as the reference for the binary inverse below.
template <class C>
FF_HD fe fe_inv_fermat(const fe& a) {
    fe e;
    // p - 2 (p is odd and its low limb is >= 2, so no borrow)
#pragma unroll
    for (int i = 0; i < 8; ++i) e.l[i] = C::mod(i);
    e.l[0] -= 2u;
    return fe_pow<C>(a, e);
}

// ---- helpers of the binary inverse: plain limb arithmetic, no modular reduction -----------------
FF_HD void limbs_shr1(uint32_t* x, uint32_t top_in) {  // x = (top_in:x) >> 1
#pragma unroll
    for (int i = 0; i < 7; ++i) x[i] = (x[i] >> 1) | (x[i + 1] << 31);
    x[7] = (x[7] >> 1) | (top_in << 31);
}
template <class C>
FF_HD uint32_t limbs_add_mod(uint32_t* x) {  // x += p, returns the carry out
    uint64_t c = 0;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        c += (uint64_t)x[i] + C::mod(i);
        x[i] = (uint32_t)c;
        c >>= 32;
    }
    return (uint32_t)c;
}
FF_HD bool limbs_ge(const uint32_t* x, const uint32_t* y) {
    for (int i = 7; i >= 0; --i)
        if (x[i] != y[i]) return x[i] > y[i];
    return true;
}
// The limbs encode an element of the field: a Montgomery residue a 2^256 mod p lies in [0, p).  Everything above maps
// to the same residue under fe_mul but not under fe_add / fe_sub, so a verifier refuses it where it enters.
template <class C>
FF_HD bool fe_is_canonical(const fe& a) {
    uint32_t m[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) m[i] = C::mod(i);
    return !limbs_ge(a.l, m);
}
FF_HD void limbs_sub(uint32_t* x, const uint32_t* y) {  // x -= y (x >= y)
    int64_t br = 0;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const int64_t d = (int64_t)x[i] - (int64_t)y[i] + br;
        x[i] = (uint32_t)d;
        br = d >> 32;
    }
}
FF_HD bool limbs_is_one(const uint32_t* x) {
    uint32_t o = x[0] ^ 1u;
#pragma unroll
    for (int i = 1; i < 8; ++i) o |= x[i];
    return o == 0;
}

// Inverse by the binary extended Euclidean algorithm (shifts and subtractions only: ~20x shorter
// dependency chain than the 380-product Fermat ladder, which matters in the latency-bound kernels).
// Input a*R, output a^-1 * R; inv(0) = 0.  Invariants: b*a == u, c*a == v (mod p).
template <class C>
FF_HD fe fe_inv_euclid(const fe& a) {
    if (fe_is_zero(a)) return fe_zero();
    uint32_t u[8], v[8];
    fe b = fe_zero(), c = fe_zero();
    b.l[0] = 1u;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        u[i] = a.l[i];
        v[i] = C::mod(i);
    }
    while (!limbs_is_one(u) && !limbs_is_one(v)) {
        while (!(u[0] & 1u)) {
            limbs_shr1(u, 0u);
            uint32_t carry = 0;
            if (b.l[0] & 1u) carry = limbs_add_mod<C>(b.l);
            limbs_shr1(b.l, carry);
        }
        while (!(v[0] & 1u)) {
            limbs_shr1(v, 0u);
            uint32_t carry = 0;
            if (c.l[0] & 1u) carry = limbs_add_mod<C>(c.l);
            limbs_shr1(c.l, carry);
        }
        if (limbs_ge(u, v)) {
            limbs_sub(u, v);
            b = fe_sub<C>(b, c);
        } else {
            limbs_sub(v, u);
            c = fe_sub<C>(c, b);
        }
    }
    const fe x = limbs_is_one(u) ? b : c;  // x * (a R) = 1  =>  x = a^-1 R^-1
    const fe r3 = fe_mul<C>(fe_r2<C>(), fe_r2<C>());  // R^3 (Montgomery product of R^2 by R^2)
    return fe_mul<C>(x, r3);                     // a^-1 R^-1 * R^3 * R^-1 = a^-1 R
}

#if !defined(__CUDA_ARCH__)
// ---- host inverse: Bernstein-Yang "safegcd" division steps, 62 at a time ------------------------------------------
// The host side inverts on every commitment batch (affine normalisation of the MSM results, on the proof's critical
// path) and ~130 times per pairing; the binary Euclid above costs ~10 us there.  Here the 2 x 2 transition matrix of 62
// division steps is computed on the low 64 bits of (f, g) alone and then applied to the full-width (f, g) and — with
// one Montgomery-style correction by a multiple of p — to the cofactors (d, e), as in Bernstein and Yang, "Fast
// constant-time gcd computation and modular inversion" (CHES 2019), variable-time form: <= 12 rounds of 5-limb
// multiply-accumulates instead of ~380 full-width shift / subtract rounds.  Numbers are five signed 62-bit limbs.
// Invariants: d * x == f, e * x == g (mod p); at g == 0, f == +-1 and d == +-x^-1.
namespace safegcd {
typedef __int128 i128;
constexpr uint64_t kM62 = ~(uint64_t)0 >> 2;
struct s62 {
    int64_t v[5];
};
struct trans {
    int64_t u, v, q, r;
};
inline int64_t divsteps_62(int64_t eta, uint64_t f0, uint64_t g0, trans* t) {
    uint64_t u = 1, v = 0, q = 0, r = 1, f = f0, g = g0;
    int i = 62;
    for (;;) {
        const int zeros = __builtin_ctzll(g | (~(uint64_t)0 << i));  // divide g by 2 while it is even (at most i times)
        g >>= zeros;
        u <<= zeros;
        v <<= zeros;
        eta -= zeros;
        i -= zeros;
        if (i == 0) break;
        if (eta < 0) {  // delta > 0 and g odd: (f, g) <- (g, -f)
            eta = -eta;
            uint64_t tmp = f;
            f = g;
            g = 0 - tmp;
            tmp = u;
            u = q;
            q = 0 - tmp;
            tmp = v;
            v = r;
            r = 0 - tmp;
        }
        g += f;  // both odd: the sum is even, the next pass shifts it
        q += u;
        r += v;
    }
    t->u = (int64_t)u;
    t->v = (int64_t)v;
    t->q = (int64_t)q;
    t->r = (int64_t)r;
    return eta;
}
// (f, g) <- (u f + v g, q f + r g) / 2^62 (exact)
inline void update_fg(s62* f, s62* g, const trans& t) {
    i128 cf = (i128)t.u * f->v[0] + (i128)t.v * g->v[0], cg = (i128)t.q * f->v[0] + (i128)t.r * g->v[0];
    cf >>= 62;
    cg >>= 62;
    for (int i = 1; i < 5; ++i) {
        cf += (i128)t.u * f->v[i] + (i128)t.v * g->v[i];
        cg += (i128)t.q * f->v[i] + (i128)t.r * g->v[i];
        f->v[i - 1] = (int64_t)((uint64_t)cf & kM62);
        g->v[i - 1] = (int64_t)((uint64_t)cg & kM62);
        cf >>= 62;
        cg >>= 62;
    }
    f->v[4] = (int64_t)cf;
    g->v[4] = (int64_t)cg;
}
// (d, e) <- (u d + v e, q d + r e) / 2^62 mod p, kept in (-2p, p)
inline void update_de(s62* d, s62* e, const trans& t, const s62& p, uint64_t p_inv62) {
    const int64_t sd = d->v[4] >> 63, se = e->v[4] >> 63;
    int64_t md = (t.u & sd) + (t.v & se), me = (t.q & sd) + (t.r & se);
    i128 cd = (i128)t.u * d->v[0] + (i128)t.v * e->v[0], ce = (i128)t.q * d->v[0] + (i128)t.r * e->v[0];
    md -= (int64_t)((p_inv62 * (uint64_t)cd + (uint64_t)md) & kM62);  // now the low 62 bits of cd + p * md vanish
    me -= (int64_t)((p_inv62 * (uint64_t)ce + (uint64_t)me) & kM62);
    cd += (i128)p.v[0] * md;
    ce += (i128)p.v[0] * me;
    cd >>= 62;
    ce >>= 62;
    for (int i = 1; i < 5; ++i) {
        cd += (i128)t.u * d->v[i] + (i128)t.v * e->v[i] + (i128)p.v[i] * md;
        ce += (i128)t.q * d->v[i] + (i128)t.r * e->v[i] + (i128)p.v[i] * me;
        d->v[i - 1] = (int64_t)((uint64_t)cd & kM62);
        e->v[i - 1] = (int64_t)((uint64_t)ce & kM62);
        cd >>= 62;
        ce >>= 62;
    }
    d->v[4] = (int64_t)cd;
    e->v[4] = (int64_t)ce;
}
inline void carry(s62* a) {  // limbs 0..3 into [0, 2^62), the sign stays in limb 4
    for (int i = 0; i < 4; ++i) {
        a->v[i + 1] += a->v[i] >> 62;
        a->v[i] &= (int64_t)kM62;
    }
}
inline s62 from_words(const uint64_t w[4]) {
    s62 r;
    r.v[0] = (int64_t)(w[0] & kM62);
    r.v[1] = (int64_t)(((w[0] >> 62) | (w[1] << 2)) & kM62);
    r.v[2] = (int64_t)(((w[1] >> 60) | (w[2] << 4)) & kM62);
    r.v[3] = (int64_t)(((w[2] >> 58) | (w[3] << 6)) & kM62);
    r.v[4] = (int64_t)(w[3] >> 56);
    return r;
}
}  // namespace safegcd

// a^-1 for a canonical residue given as 8 limbs (plain integers in, plain integer out); false if no inverse was reached
template <class C>
inline bool limbs_inv_safegcd(const uint32_t a[8], uint32_t out[8]) {
    using namespace safegcd;
    uint64_t pw[4], xw[4];
    for (int i = 0; i < 4; ++i) {
        pw[i] = (uint64_t)C::mod(2 * i) | ((uint64_t)C::mod(2 * i + 1) << 32);
        xw[i] = (uint64_t)a[2 * i] | ((uint64_t)a[2 * i + 1] << 32);
    }
    uint64_t pinv = (uint64_t)(0u - C::inv);  // p^-1 mod 2^32 (C::inv is -p^-1), two Newton steps to 2^64
    pinv *= 2 - pw[0] * pinv;
    pinv *= 2 - pw[0] * pinv;
    const uint64_t p_inv62 = pinv & kM62;
    const s62 p = from_words(pw);
    s62 f = p, g = from_words(xw), d = {{0, 0, 0, 0, 0}}, e = {{1, 0, 0, 0, 0}};
    int64_t eta = -1;
    bool done = false;
    for (int round = 0; round < 14 && !done; ++round) {  // <= 12 rounds of 62 steps cover 256-bit inputs
        trans t;
        eta = divsteps_62(eta, (uint64_t)f.v[0], (uint64_t)g.v[0], &t);
        update_de(&d, &e, t, p, p_inv62);
        update_fg(&f, &g, t);
        done = (g.v[0] | g.v[1] | g.v[2] | g.v[3] | g.v[4]) == 0;
    }
    if (!done) return false;
    // f == +-1; the inverse is d with f's sign, brought into [0, p)
    const bool f_neg = f.v[4] < 0;
    if (!((f.v[0] == 1 && !f.v[1] && !f.v[2] && !f.v[3] && !f.v[4]) ||
          (f_neg && f.v[0] == (int64_t)kM62 && f.v[1] == (int64_t)kM62 && f.v[2] == (int64_t)kM62 && f.v[3] == (int64_t)kM62 && f.v[4] == -1)))
        return false;  // gcd(x, p) != 1 (x == 0)
    if (f_neg)
        for (int i = 0; i < 5; ++i) d.v[i] = -d.v[i];
    carry(&d);
    for (int k = 0; k < 3 && d.v[4] < 0; ++k) {
        for (int i = 0; i < 5; ++i) d.v[i] += p.v[i];
        carry(&d);
    }
    for (int k = 0; k < 3; ++k) {  // while d >= p: subtract
        s62 tmp = d;
        for (int i = 0; i < 5; ++i) tmp.v[i] -= p.v[i];
        carry(&tmp);
        if (tmp.v[4] < 0) break;
        d = tmp;
    }
    const uint64_t w0 = (uint64_t)d.v[0] | ((uint64_t)d.v[1] << 62), w1 = ((uint64_t)d.v[1] >> 2) | ((uint64_t)d.v[2] << 60),
                   w2 = ((uint64_t)d.v[2] >> 4) | ((uint64_t)d.v[3] << 58), w3 = ((uint64_t)d.v[3] >> 6) | ((uint64_t)d.v[4] << 56);
    const uint64_t w[4] = {w0, w1, w2, w3};
    for (int i = 0; i < 4; ++i) {
        out[2 * i] = (uint32_t)w[i];
        out[2 * i + 1] = (uint32_t)(w[i] >> 32);
    }
    return true;
}

// Montgomery in, Montgomery out: inv(a R) = a^-1 R^-1, times R^3 by one Montgomery product
template <class C>
inline fe fe_inv_safegcd(const fe& a) {
    if (fe_is_zero(a)) return fe_zero();
    fe x;
    if (!limbs_inv_safegcd<C>(a.l, x.l)) return fe_inv_euclid<C>(a);
    return fe_mul<C>(x, fe_mul<C>(fe_r2<C>(), fe_r2<C>()));
}
#endif

template <class C>
FF_HD fe fe_inv(const fe& a) {
#if defined(__CUDA_ARCH__)
    // When every lane of a warp inverts its own element the data-dependent branches of the binary algorithm diverge
    // (measured slower than the branch-free ladder), so per-thread inversions keep Fermat; a kernel that
    // needs ONE inversion calls fe_inv_euclid from a single lane.
    return fe_inv_fermat<C>(a);
#else
    return fe_inv_safegcd<C>(a);  // ~1.5 us; the binary Euclid (~10 us) stays as its fallback and as the device's one-lane inverse
#endif
}

// small-integer constant in Montgomery form
template <class C>
FF_HD fe fe_from_u32(uint32_t v) {
    fe x = fe_zero();
    x.l[0] = v;
    return fe_to_mont<C>(x);
}

// ---------------------------------------------------------------------------------------------
// 128-bit global-memory access: one element = two uint4 (one 32-byte sector)
// ---------------------------------------------------------------------------------------------
#if defined(__CUDACC__)
FF_D fe fe_load(const fe* p) {
    const uint4* q = reinterpret_cast<const uint4*>(p);
    uint4 lo = q[0], hi = q[1];
    fe r;
    r.l[0] = lo.x; r.l[1] = lo.y; r.l[2] = lo.z; r.l[3] = lo.w;
    r.l[4] = hi.x; r.l[5] = hi.y; r.l[6] = hi.z; r.l[7] = hi.w;
    return r;
}
FF_D fe fe_load_ro(const fe* p) {  // read-only path (twiddles, bases)
    const uint4* q = reinterpret_cast<const uint4*>(p);
    uint4 lo = __ldg(q), hi = __ldg(q + 1);
    fe r;
    r.l[0] = lo.x; r.l[1] = lo.y; r.l[2] = lo.z; r.l[3] = lo.w;
    r.l[4] = hi.x; r.l[5] = hi.y; r.l[6] = hi.z; r.l[7] = hi.w;
    return r;
}
FF_D void fe_store(fe* p, const fe& v) {
    uint4* q = reinterpret_cast<uint4*>(p);
    q[0] = make_uint4(v.l[0], v.l[1], v.l[2], v.l[3]);
    q[1] = make_uint4(v.l[4], v.l[5], v.l[6], v.l[7]);
}
#endif

}  // namespace b200
