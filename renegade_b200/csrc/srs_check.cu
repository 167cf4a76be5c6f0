// Consistency check of a loaded SRS: are the n G1 powers P_i = tau^i P_0 for the tau of the G2 pair (h, beta_h = tau h),
// is P_0 the generator G = (1, 2) the verifiers use, and are h and beta_h of order r?
//
// The reference samples 100 of the consecutive pairs with e(P_i, tau H) == e(P_{i+1}, H) in a unit test
// (circuit-types/src/primitives/srs.rs:251-266) and otherwise relies on `snarkjs powersoftau verify`.  Here every pair
// is covered at once by a random linear combination with the powers of one rho:
//     A = sum_{i < n-1} rho^i P_i,   B = sum_{i < n-1} rho^i P_{i+1},   e(A, tau H) == e(B, H).
// If some pair fails, A - tau B is a non-zero polynomial of degree < n - 1 in rho, so the check passes with probability
// at most n / r over a rho the file's maker cannot predict.  A and B are ONE batch-2 MSM over the resident bases
// (msm_device_batch, the MSM behind b200_msm_batch_device), the weights come from k_srs_weights, and the 2-pair pairing
// runs on the host (pairing_two_is_one, verify.cu).  When it fails and the caller asks where, k_srs_pairs checks every
// pair on its own on the device (pairing.cuh, one thread per pair), reading the points where the MSM reads them.
// The G2 subgroup test, [r]Q == O, runs on the host in Jacobian coordinates: two scalar multiplications per check.
#include <cstring>
#include <mutex>
#include <string>
#include <vector>

#include "b200prover.h"
#include "device_ctx.h"
#include "pairing.cuh"
#include "transcript.h"
#include "verify_terms.h"

namespace b200 {

namespace {

using Fr = FrCfg;

// rho^(2^k), k < kRhoBits: a thread's first weight rho^start from the bits of start
constexpr int kRhoBits = 48;
struct RhoPowers {
    fe p[kRhoBits];
};
constexpr int kWeightChunk = 32;  // weights per thread: one product per element after the first
constexpr int kWeightThreads = 128;

// s[0, n): s_A[i] = rho^i (i < n - 1), s_A[n - 1] = 0;  s[n, 2n): s_B[0] = 0, s_B[i] = rho^(i-1).  Montgomery form.
__global__ void __launch_bounds__(kWeightThreads) k_srs_weights(RhoPowers rp, size_t n, fe* __restrict__ s) {
    const size_t start = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) * kWeightChunk;
    if (start >= n) return;
    fe* sa = s;
    fe* sb = s + n;
    if (start == 0) {
        fe_store(sa + (n - 1), fe_zero());
        fe_store(sb, fe_zero());
    }
    fe v = fe_one<Fr>();
    for (int k = 0; k < kRhoBits; ++k)
        if ((start >> k) & 1) v = fe_mul<Fr>(v, rp.p[k]);
    const size_t end = start + kWeightChunk < n - 1 ? start + kWeightChunk : n - 1;
    for (size_t i = start; i < end; ++i) {
        fe_store(sa + i, v);
        fe_store(sb + i + 1, v);
        v = fe_mul<Fr>(v, rp.p[0]);
    }
}

// ok[i] = [ e(P_i, tau H) * e(-P_{i+1}, H) == 1 ] for the n_pairs consecutive pairs of pts, q = the prepared lines of
// (tau H, H); a pair with a point off the curve (or a coordinate >= q) fails.
constexpr int kSrsPairThreads = 64;
__global__ void __launch_bounds__(kSrsPairThreads) k_srs_pairs(const G2Prepared* __restrict__ q, const g1_affine* __restrict__ pts,
                                                               size_t n_pairs, PairingConsts pc, uint8_t* __restrict__ ok) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_pairs) return;
    const g1_affine a = pts[i], b = pts[i + 1];
    if (!g1_affine_on_curve(a) || !g1_affine_on_curve(b)) {
        ok[i] = 0;
        return;
    }
    const g1_affine p[2] = {a, g1_affine_neg(b)};
    ok[i] = fq12_is_one(final_exponentiation(miller_loop_prepared(q, p, 2), pc)) ? 1 : 0;
}

// ---- G2 on the host, Jacobian coordinates (x = X / Z^2, y = Y / Z^3; Z = 0 is the identity) ---------------------------
struct g2_jac {
    fq2 x, y, z;
};
// 2P (EFD dbl-2009-l, a = 0); a point with y = 0 doubles to the identity through Z3 = 2 Y Z
g2_jac g2_jac_dbl(const g2_jac& p) {
    const fq2 a = fq2_sqr(p.x), b = fq2_sqr(p.y), c = fq2_sqr(b);
    fq2 d = fq2_sub(fq2_sub(fq2_sqr(fq2_add(p.x, b)), a), c);
    d = fq2_add(d, d);
    const fq2 e = fq2_add(fq2_add(a, a), a);
    const fq2 f = fq2_sqr(e);
    g2_jac r;
    r.x = fq2_sub(f, fq2_add(d, d));
    fq2 c8 = fq2_add(c, c);
    c8 = fq2_add(c8, c8);
    c8 = fq2_add(c8, c8);
    r.y = fq2_sub(fq2_mul(e, fq2_sub(d, r.x)), c8);
    const fq2 yz = fq2_mul(p.y, p.z);
    r.z = fq2_add(yz, yz);
    return r;
}
// P + Q, Q affine and not the identity (EFD madd-2007-bl), with P == Q and P == -Q handled exactly
g2_jac g2_jac_add_affine(const g2_jac& p, const g2_affine& q) {
    if (fq2_is_zero(p.z)) return {q.x, q.y, {fe_one<Fq>(), fe_zero()}};
    const fq2 z1z1 = fq2_sqr(p.z);
    const fq2 u2 = fq2_mul(q.x, z1z1);
    const fq2 s2 = fq2_mul(q.y, fq2_mul(p.z, z1z1));
    const fq2 h = fq2_sub(u2, p.x);
    fq2 rr = fq2_sub(s2, p.y);
    if (fq2_is_zero(h)) {
        if (fq2_is_zero(rr)) return g2_jac_dbl(p);
        return {{fe_one<Fq>(), fe_zero()}, {fe_one<Fq>(), fe_zero()}, {fe_zero(), fe_zero()}};
    }
    rr = fq2_add(rr, rr);
    const fq2 hh = fq2_sqr(h);
    fq2 i = fq2_add(hh, hh);
    i = fq2_add(i, i);
    const fq2 j = fq2_mul(h, i);
    const fq2 v = fq2_mul(p.x, i);
    g2_jac r;
    r.x = fq2_sub(fq2_sub(fq2_sqr(rr), j), fq2_add(v, v));
    const fq2 y1j = fq2_mul(p.y, j);
    r.y = fq2_sub(fq2_mul(rr, fq2_sub(v, r.x)), fq2_add(y1j, y1j));
    r.z = fq2_sub(fq2_sub(fq2_sqr(fq2_add(p.z, h)), z1z1), hh);
    return r;
}
// [r]Q == O by double-and-add over the bits of r; the identity is not in the subgroup here
bool g2_in_subgroup(const g2_affine& q) {
    if (q.inf) return false;
    g2_jac acc = {{fe_one<Fq>(), fe_zero()}, {fe_one<Fq>(), fe_zero()}, {fe_zero(), fe_zero()}};
    for (int bit = 255; bit >= 0; --bit) {
        acc = g2_jac_dbl(acc);
        if ((Fr::mod(bit >> 5) >> (bit & 31)) & 1u) acc = g2_jac_add_affine(acc, q);
    }
    return fq2_is_zero(acc.z);
}

// rho = keccak256("b200 srs check v1" || seed || n as u64 big-endian || g2_h || g2_tau_h) as a big-endian integer mod r
// (1 if that is 0), Montgomery form
fe srs_rho(const uint8_t seed[32], size_t n, const uint64_t g2_h[16], const uint64_t g2_tau_h[16]) {
    static const char tag[] = "b200 srs check v1";
    uint8_t h[32], be[8];
    for (int b = 0; b < 8; ++b) be[b] = (uint8_t)((uint64_t)n >> (56 - 8 * b));
    Keccak256 kc;
    kc.absorb(reinterpret_cast<const uint8_t*>(tag), sizeof(tag) - 1);
    kc.absorb(seed, 32);
    kc.absorb(be, 8);
    kc.absorb(reinterpret_cast<const uint8_t*>(g2_h), 128);
    kc.absorb(reinterpret_cast<const uint8_t*>(g2_tau_h), 128);
    kc.finish(h);
    fe rho = fe_zero();
    const fe c256 = fe_from_u32<Fr>(256);
    for (int b = 0; b < 32; ++b) rho = fe_add<Fr>(fe_mul<Fr>(rho, c256), fe_from_u32<Fr>(h[b]));
    return fe_is_zero(rho) ? fe_one<Fr>() : rho;
}

inline unsigned grid_of(size_t n, unsigned bs) { return (unsigned)((n + bs - 1) / bs); }

// the combined check over bases[0, n), n >= 2; caller holds the context's lock
int combined_check(Context* c, const Bases* b, size_t n, const uint64_t g2_h[16], const uint64_t g2_tau_h[16],
                   const fe& rho, bool* ok) {
    cudaStream_t st = c->stream;
    RhoPowers rp;
    rp.p[0] = rho;
    for (int k = 1; k < kRhoBits; ++k) rp.p[k] = fe_sqr<Fr>(rp.p[k - 1]);
    DevBuf d_s;
    int rc = d_s.reserve(2 * n * sizeof(fe));
    if (rc != B200_OK) return rc;
    B200_LAUNCH(k_srs_weights, grid_of(grid_of(n, kWeightChunk), kWeightThreads), kWeightThreads, 0, st)(rp, n, (fe*)d_s.p);
    B200_CUDA(cudaGetLastError());
    g1_affine out[2];
    int inf[2];
    if ((rc = msm_device_batch(b, 0, (const fe*)d_s.p, n, n, 2, 1, &c->msm, st, out, inf)) != B200_OK) return rc;
    for (int j = 0; j < 2; ++j)
        if (inf[j]) out[j].x = out[j].y = fe_zero();
    return pairing_two_is_one(out[0], g1_affine_neg(out[1]), g2_tau_h, g2_h, ok);
}

// every consecutive pair of bases[0, n) on its own; fills n_bad / bad; caller holds the context's lock
int locate_pairs(Context* c, const Bases* b, size_t n, const uint64_t g2_h[16], const uint64_t g2_tau_h[16],
                 b200_srs_report* out) {
    cudaStream_t st = c->stream;
    const size_t n_pairs = n - 1;
    std::vector<G2Prepared> q(2);  // (tau H, H), both on the curve (checked by the caller)
    g2_prepare_record(g2_tau_h, &q[0]);
    g2_prepare_record(g2_h, &q[1]);
    DevBuf d_q, d_ok;
    int rc;
    if ((rc = d_q.reserve(q.size() * sizeof(G2Prepared))) != B200_OK || (rc = d_ok.reserve(n_pairs)) != B200_OK) return rc;
    B200_CUDA(cudaMemcpyAsync(d_q.p, q.data(), q.size() * sizeof(G2Prepared), cudaMemcpyHostToDevice, st));
    // table 0 of the bases is the points themselves
    B200_LAUNCH(k_srs_pairs, grid_of(n_pairs, kSrsPairThreads), kSrsPairThreads, 0, st)(
        (const G2Prepared*)d_q.p, b->tables, n_pairs, pairing_consts(), (uint8_t*)d_ok.p);
    B200_CUDA(cudaGetLastError());
    std::vector<uint8_t> ok(n_pairs);
    B200_CUDA(cudaMemcpyAsync(ok.data(), d_ok.p, n_pairs, cudaMemcpyDeviceToHost, st));
    B200_CUDA(cudaStreamSynchronize(st));
    for (size_t i = 0; i < n_pairs; ++i) {
        if (ok[i]) continue;
        if (out->n_bad < 8) out->bad[out->n_bad] = i;
        ++out->n_bad;
    }
    return B200_OK;
}

}  // namespace

}  // namespace b200

using namespace b200;

extern "C" {

int b200_g2_in_subgroup(const uint64_t rec[16], int* in_subgroup) {
    B200_TRY
    if (!rec || !in_subgroup) return B200_ERR_INVALID;
    g2_affine q;
    if (!g2_load_record(rec, &q)) {
        set_error("g2_in_subgroup: G2 point not on curve");
        return B200_ERR_NOT_ON_CURVE;
    }
    *in_subgroup = g2_in_subgroup(q) ? 1 : 0;
    return B200_OK;
    B200_CATCH
}

int b200_srs_check(b200_ctx* ctx, const b200_bases* srs, size_t n, const uint64_t g2_h[16], const uint64_t g2_tau_h[16],
                   const uint8_t seed[32], int locate, b200_srs_report* out) {
    B200_TRY
    if (!ctx || !srs || !g2_h || !g2_tau_h || !seed || !out) return B200_ERR_INVALID;
    if (n == 0 || n > srs->b->n) {
        set_error("srs_check: n must be in [1, " + std::to_string(srs->b->n) + "]");
        return B200_ERR_INVALID;
    }
    if (n >= ((size_t)1 << kRhoBits)) {
        set_error("srs_check: n >= 2^48");
        return B200_ERR_INVALID;
    }
    g2_affine h, tau_h;
    if (!g2_load_record(g2_h, &h) || !g2_load_record(g2_tau_h, &tau_h)) {
        set_error("srs_check: G2 point not on curve");
        return B200_ERR_NOT_ON_CURVE;
    }
    b200_srs_report r;
    std::memset(&r, 0, sizeof(r));
    r.g2_subgroup = g2_in_subgroup(h) && g2_in_subgroup(tau_h) ? 1 : 0;
    const fe rho = srs_rho(seed, n, g2_h, g2_tau_h);
    std::lock_guard<std::mutex> lk(ctx->c.mu);
    B200_ENTER(ctx->c);
    cudaStream_t st = ctx->c.stream;
    g1_affine p0;
    B200_CUDA(cudaMemcpyAsync(&p0, srs->b->tables, sizeof(p0), cudaMemcpyDeviceToHost, st));
    B200_CUDA(cudaStreamSynchronize(st));
    const g1_affine g = vt::g1_generator();
    r.g1_generator = fe_eq(p0.x, g.x) && fe_eq(p0.y, g.y) ? 1 : 0;
    r.consistent = 1;
    if (n >= 2) {
        bool ok = false;
        int rc = combined_check(&ctx->c, srs->b, n, g2_h, g2_tau_h, rho, &ok);
        if (rc != B200_OK) return rc;
        r.consistent = ok ? 1 : 0;
        if (!ok && locate && (rc = locate_pairs(&ctx->c, srs->b, n, g2_h, g2_tau_h, &r)) != B200_OK) return rc;
    }
    *out = r;
    return B200_OK;
    B200_CATCH
}

}  // extern "C"
