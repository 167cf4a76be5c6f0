// b200_selftest_pairing: seeded operands through the group arithmetic of pairing_warp.cuh and through the one-thread
// functions of pairing.cuh on the device.  One 16-lane group per iteration; every lane also runs the one-thread
// function and lane j compares coefficient j, so a result counts once when any of its 12 coefficients differs.
#include <cstring>
#include <mutex>
#include <vector>

#include "b200prover.h"
#include "b200selftest.h"
#include "device_ctx.h"
#include "pairing.cuh"
#include "pairing_warp.cuh"

namespace b200 {
namespace {

FF_D uint64_t splitmix(uint64_t seed, uint64_t j) {
    uint64_t z = seed + (j + 1) * 0x9E3779B97F4A7C15ULL;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ULL;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBULL;
    return z ^ (z >> 31);
}
// Uniform on [0, q): 254-bit draws (q > 2^253, so about 3 in 4 are accepted), the next draw while one is not below q
FF_D fe random_fe(uint64_t seed, uint64_t i) {
    fe v;
    for (uint64_t t = 0;; ++t) {
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const uint64_t x = splitmix(seed + t * 0x632BE59BD9B4E019ULL, 4 * i + k);
            v.l[2 * k] = (uint32_t)x;
            v.l[2 * k + 1] = (uint32_t)(x >> 32);
        }
        v.l[7] &= 0x3fffffffu;
        if (fe_is_canonical<FqCfg>(v)) return v;
    }
}
// The values at the top and the middle of Fq and at the powers of two a reduction meets: q - 1, (q - 1) / 2,
// R mod q (the Montgomery one) and 2^252
FF_D fe edge_fe(int e) {
    fe v = fe_zero();
    if (e == 0 || e == 1) {
#pragma unroll
        for (int k = 0; k < 8; ++k) v.l[k] = FqCfg::mod(k);
        v.l[0] -= 1;  // q is odd
        if (e == 1)
#pragma unroll
            for (int k = 0; k < 8; ++k) v.l[k] = (v.l[k] >> 1) | (k < 7 ? v.l[k + 1] << 31 : 0u);
    } else if (e == 2) {
#pragma unroll
        for (int k = 0; k < 8; ++k) v.l[k] = FqCfg::one(k);
    } else {
        v.l[7] = 1u << 28;
    }
    return v;
}
// Operand o of iteration i.  The shapes cycle so that every operation meets dense values, values with about half their
// coefficients zero, the value 1, elements of Fq2 = Fq + Fq w^6 (the inversion's last step), 0, values made only of the
// edge values of edge_fe, and dense values with about half their coefficients edge values.
FF_D fq12 random_fq12(uint64_t seed, uint64_t i, int o) {
    const int shape = (int)((i + o) % 8);
    const uint64_t zeros = splitmix(seed ^ 0x2e705ULL, 2 * i + o);
    fq12 a;
#pragma unroll
    for (int k = 0; k < 12; ++k) {
        a.c[k] = random_fe(seed, (2 * i + o) * 12 + k);
        if ((shape == 2 && ((zeros >> k) & 1)) || (shape == 4 && k % 6) || shape == 5) a.c[k] = fe_zero();
        if (shape == 6 || (shape == 7 && ((zeros >> k) & 1))) a.c[k] = edge_fe((int)((zeros >> (16 + 2 * k)) & 3));
    }
    return shape == 3 ? fq12_one() : a;
}
FF_D fe coeff(const fq12& a, int j) {
    fe r = a.c[0];
#pragma unroll
    for (int k = 1; k < 12; ++k)
        if (j == k) r = a.c[k];
    return r;
}
// 1 when the group's coefficients differ from ref's anywhere, on every lane of the group
FF_D unsigned differs(const fe& mine, const fq12& ref) {
    const pw::Lanes g = pw::lanes();
    const bool ok = fe_eq(mine, coeff(ref, g.j));
    return (__ballot_sync(g.mask, !ok) & g.mask) ? 1u : 0u;
}

constexpr int kSelftestThreads = 128;
// q: two prepared G2 points for the Miller loop
__global__ void __launch_bounds__(kSelftestThreads) k_selftest_pairing(uint64_t seed, size_t iters,
                                                                       const G2Prepared* __restrict__ q, PairingConsts pc,
                                                                       unsigned long long* bad) {
    __shared__ pw::Consts kc;
    if (threadIdx.x == 0) pw::consts_init(&kc, pc);
    __syncthreads();
    const size_t i = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) / pw::kGroup;
    if (i >= iters) return;
    const pw::Lanes g = pw::lanes();
    const fq12 a = random_fq12(seed, i, 0), b = random_fq12(seed, i, 1);
    const fe aj = coeff(a, g.j), bj = coeff(b, g.j);
    unsigned n = 0;
    n += differs(pw::mul(aj, bj, &kc), fq12_mul(a, b));
    n += differs(pw::sqr(aj, &kc), fq12_sqr(a));
    // a line of every kind (none, vertical, sloped) with random coefficients, at a random point
    G2Line l;
    l.kind = (uint32_t)(i % 3);
    l.a = {random_fe(seed ^ 0x11, 4 * i), random_fe(seed ^ 0x11, 4 * i + 1)};
    l.b = {random_fe(seed ^ 0x11, 4 * i + 2), random_fe(seed ^ 0x11, 4 * i + 3)};
    const fe px = random_fe(seed ^ 0x22, 2 * i), py = random_fe(seed ^ 0x22, 2 * i + 1);
    fq12 r = a;
    line_eval_mul(&r, l, px, py);
    n += differs(pw::line_mul(aj, &l, px, py, &kc), r);
    n += differs(pw::conj(aj), fq12_conj(a));
    n += differs(pw::frob1(aj, &kc), fq12_frob1(a, pc));
    n += differs(pw::frob2(aj, &kc), fq12_frob2(a, pc));
    n += differs(pw::inv(aj, &kc), fq12_inv(a));
    n += differs(pw::pow_x(aj, &kc), fq12_pow_x(a));
    n += differs(pw::final_exp(aj, &kc), final_exponentiation(a, pc));
    // the Miller loop over both prepared points; the G1 coordinates are random (the loop is algebraic in them), and
    // either point is the identity now and then
    g1_affine p[2];
    for (int o = 0; o < 2; ++o) {
        p[o].x = random_fe(seed ^ 0x33, 4 * i + 2 * o);
        p[o].y = random_fe(seed ^ 0x33, 4 * i + 2 * o + 1);
        if (i % 5 == (uint64_t)o + 1) p[o].x = p[o].y = fe_zero();
    }
    const unsigned skip = (g1_affine_is_inf(p[0]) ? 1u : 0u) | (g1_affine_is_inf(p[1]) ? 2u : 0u);
    const fe xj = g.lane == 1 ? p[1].x : p[0].x, yj = g.lane == 1 ? p[1].y : p[0].y;
    n += differs(pw::miller(q, 2, xj, yj, skip, &kc), miller_loop_prepared(q, p, 2));
    if (g.lane == 0 && n) atomicAdd(bad, (unsigned long long)n);
}

// The BN254 G2 generator (x0, x1, y0, y1), canonical little-endian limbs
constexpr uint64_t kG2Gen[16] = {
    0x46debd5cd992f6edULL, 0x674322d4f75edaddULL, 0x426a00665e5c4479ULL, 0x1800deef121f1e76ULL,
    0x97e485b7aef312c2ULL, 0xf1aa493335a9e712ULL, 0x7260bfb731fb5d25ULL, 0x198e9393920d483aULL,
    0x4ce6cc0166fa7daaULL, 0xe3d1e7690c43d37bULL, 0x4aab71808dcb408fULL, 0x12c85ea5db8c6debULL,
    0x55acdadcd122975bULL, 0xbc4b313370b38ef3ULL, 0xec9e99ad690c3395ULL, 0x090689d0585ff075ULL};

}  // namespace
}  // namespace b200

using namespace b200;

extern "C" int b200_selftest_pairing(b200_ctx* ctx, uint64_t seed, size_t iters, uint64_t* mismatches) {
    B200_TRY
    int count = 0;
    if (cudaGetDeviceCount(&count) != cudaSuccess || count == 0) {
        set_error("selftest_pairing: no CUDA device (libb200prover has no CPU fallback)");
        return B200_ERR_NO_DEVICE;
    }
    if (!ctx || !mismatches) return B200_ERR_INVALID;
    // the Miller loop's points: the G2 generator H and -H, prepared on the host like a verifier's pair
    uint64_t rec[2][16];
    for (int c = 0; c < 4; ++c) {
        fe v;
        std::memcpy(&v, kG2Gen + 4 * c, sizeof(fe));
        v = fe_to_mont<FqCfg>(v);
        std::memcpy(rec[0] + 4 * c, &v, sizeof(fe));
        if (c >= 2) v = fe_neg<FqCfg>(v);
        std::memcpy(rec[1] + 4 * c, &v, sizeof(fe));
    }
    std::vector<G2Prepared> q(2);
    if (!g2_prepare_record(rec[0], &q[0]) || !g2_prepare_record(rec[1], &q[1])) {
        set_error("selftest_pairing: the G2 generator is off the curve");
        return B200_ERR_INVALID;
    }
    std::lock_guard<std::mutex> lk(ctx->c.mu);
    B200_ENTER(ctx->c);
    cudaStream_t st = ctx->c.stream;
    DevBuf d_q, d_bad;
    int rc;
    if ((rc = d_q.reserve(q.size() * sizeof(G2Prepared))) || (rc = d_bad.reserve(8))) return rc;
    B200_CUDA(cudaMemcpyAsync(d_q.p, q.data(), q.size() * sizeof(G2Prepared), cudaMemcpyHostToDevice, st));
    B200_CUDA(cudaMemsetAsync(d_bad.p, 0, 8, st));
    if (iters)
        B200_LAUNCH(k_selftest_pairing, (unsigned)((iters * pw::kGroup + kSelftestThreads - 1) / kSelftestThreads),
                    kSelftestThreads, 0, st)(seed, iters, (const G2Prepared*)d_q.p, pairing_consts(),
                                             (unsigned long long*)d_bad.p);
    B200_CUDA(cudaGetLastError());
    unsigned long long h = 0;
    B200_CUDA(cudaMemcpyAsync(&h, d_bad.p, 8, cudaMemcpyDeviceToHost, st));
    B200_CUDA(cudaStreamSynchronize(st));
    *mismatches = h;
    return B200_OK;
    B200_CATCH
}
