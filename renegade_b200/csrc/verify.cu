// Host-side verifier of libb200prover: TurboPlonk / KZG proof verification, link-proof verification and the
// BN254 optimal-ate pairing they end in.  No device work: in the reference, too, verification stays on the
// CPU (SURVEY.md §8(a) a10).  The A / B terms of both checks are built by verify_terms.h, which the batch verifier
// (verify_batch.cu) runs on the device; the pairing here also ends every batch.
//
// Replaces what the reference reaches through
//   `SingleProverCircuit::verify` -> `PlonkKzgSnark::<Bn254>::verify::<SolidityTranscript>(&vk, &statement
//     scalars, &proof, None)` (/root/reference/crates/circuits/circuit-types/src/traits.rs:1003-1019), and
//   `validate_*_link` -> `PlonkKzgSnark::verify_link_proof` (circuits-core/src/zk_circuits/proof_linking/
//     intent_only.rs:54-85),
// and the pairing of the reference's own SRS unit test (circuit-types/src/primitives/srs.rs:236-266:
// e(tau^i G, tau H) == e(tau^(i+1) G, H)).  The upstream code (mpc-jellyfish `verifier.rs`, ark-ec's bn
// pairing) is not vendored; what is restated here is the published algorithm:
//   * verifier: recompute the six challenges from the transcript, evaluate Z_H, L_1 and the public-input
//     polynomial at zeta, assemble the linearisation commitment D, the batched commitment F and evaluation E,
//     and check   e(W_z + u W_zw, [tau]_2) == e(zeta W_z + u zeta w W_zw + F - E G + u ([z] - z_w G), [1]_2);
//   * pairing: pairing.cuh, the code the device pairing checks run too; here the host side of it: the Frobenius
//     constants and the preparation of G2 points (the lines of their Miller loop by affine steps).
// Clarity first: flat Fq12 arithmetic, affine Miller steps; a verification is ~6 ms of host time.
#include <cstring>
#include <mutex>
#include <vector>

#include "b200prover.h"
#include "device_ctx.h"
#include "pairing.cuh"
#include "transcript.h"
#include "verify_terms.h"

namespace b200 {

const PairingConsts& pairing_consts() {
    static PairingConsts pc;
    static std::once_flag once;
    std::call_once(once, [] {
        // q^2 - 1, little-endian limbs
        static const uint64_t q2m1[8] = {0x3b5458a2275d69b0ULL, 0xa602072d09eac101ULL, 0x4a50189c6d96cadcULL, 0x04689e957a1242c8ULL,
                                         0x26edfa5c34c6b38dULL, 0xb00b855116375606ULL, 0x599a6f7c0348d21cULL, 0x0925c4b8763cbf9cULL};
        fq12 w;
        for (auto& v : w.c) v = fe_zero();
        w.c[1] = fe_one<Fq>();
        const fq12 g = fq12_pow(w, q2m1, 8);  // w^(q^2 - 1) = gamma, an element of Fq: w^(q^2) = gamma w
        pc.gamma_pow[0] = fe_one<Fq>();
        pc.gamma_pow[1] = g.c[0];
        for (int k = 2; k < 6; ++k) pc.gamma_pow[k] = fe_mul<Fq>(pc.gamma_pow[k - 1], pc.gamma_pow[1]);
        // (q - 1) / 3 and (q - 1) / 2 from the modulus limbs
        uint64_t qm1[4];
        for (int i = 0; i < 4; ++i) qm1[i] = (uint64_t)Fq::mod(2 * i) | ((uint64_t)Fq::mod(2 * i + 1) << 32);
        qm1[0] -= 1;  // q is odd: no borrow
        uint64_t third[4], halfe[4];
        unsigned __int128 rem = 0;
        for (int i = 3; i >= 0; --i) {
            const unsigned __int128 cur = (rem << 64) | qm1[i];
            third[i] = (uint64_t)(cur / 3);
            rem = cur % 3;
        }
        for (int i = 0; i < 4; ++i) halfe[i] = (qm1[i] >> 1) | (i < 3 ? qm1[i + 1] << 63 : 0);
        const fq2 xi = {fe_from_u32<Fq>(9), fe_one<Fq>()};
        pc.twist_frob_x = fq2_pow(xi, third, 4);
        pc.twist_frob_y = fq2_pow(xi, halfe, 4);
        uint64_t sixth[4];  // (q - 1) / 6 = ((q - 1) / 3) / 2
        for (int i = 0; i < 4; ++i) sixth[i] = (third[i] >> 1) | (i < 3 ? third[i + 1] << 63 : 0);
        pc.frob1[0] = {fe_one<Fq>(), fe_zero()};
        pc.frob1[1] = fq2_pow(xi, sixth, 4);
        for (int k = 2; k < 12; ++k) pc.frob1[k] = fq2_mul(pc.frob1[k - 1], pc.frob1[1]);
    });
    return pc;
}

namespace {

using Fq = FqCfg;
using Fr = FrCfg;

g2_affine g2_frobenius(const g2_affine& p) {
    const PairingConsts& pc = pairing_consts();
    g2_affine r;
    r.inf = p.inf;
    r.x = fq2_mul(fq2{p.x.a, fe_neg<Fq>(p.x.b)}, pc.twist_frob_x);
    r.y = fq2_mul(fq2{p.y.a, fe_neg<Fq>(p.y.b)}, pc.twist_frob_y);
    return r;
}

// One affine Miller step: the line through r and s (the tangent when r == s), before it is evaluated at a G1 point, and
// r <- r + s
G2Line line_step(g2_affine* r, const g2_affine& s) {
    G2Line l;
    l.kind = kLineNone;
    l.a = l.b = fq2{fe_zero(), fe_zero()};
    if (r->inf || s.inf) {  // not reached for points of prime order inside the loop bounds
        if (r->inf) *r = s;
        return l;
    }
    fq2 m;
    if (fq2_eq(r->x, s.x)) {
        if (!fq2_eq(r->y, s.y) || fq2_is_zero(r->y)) {  // vertical line x_P - x_R w^2
            l.kind = kLineVertical;
            l.a = fq2_neg(r->x);
            r->inf = true;
            return l;
        }
        const fq2 xx = fq2_sqr(r->x);
        m = fq2_mul(fq2_add(fq2_add(xx, xx), xx), fq2_inv(fq2_add(r->y, r->y)));
    } else {
        m = fq2_mul(fq2_sub(s.y, r->y), fq2_inv(fq2_sub(s.x, r->x)));
    }
    l.kind = kLineSloped;
    l.a = m;
    l.b = fq2_sub(r->y, fq2_mul(m, r->x));
    const fq2 nx = fq2_sub(fq2_sub(fq2_sqr(m), r->x), s.x);
    const fq2 ny = fq2_sub(fq2_mul(m, fq2_sub(r->x, nx)), r->y);
    r->x = nx;
    r->y = ny;
    return l;
}

// Product of the Miller functions of k pairs (P_i in G1, Q_i in G2) before the final exponentiation: the G2 points are
// prepared, then miller_loop_prepared (pairing.cuh) evaluates their lines, the code the device pairing runs too
fq12 miller_loop_product(const g1_affine* ps, const g2_affine* qs, size_t k) {
    std::vector<g1_affine> p;
    std::vector<G2Prepared> q;
    for (size_t i = 0; i < k; ++i)
        if (!g1_affine_is_inf(ps[i]) && !qs[i].inf) {  // a pair with an identity contributes 1
            p.push_back(ps[i]);
            q.emplace_back();
            g2_prepare(qs[i], &q.back());
        }
    return miller_loop_prepared(q.data(), p.data(), (int)p.size());
}

// false for a coordinate outside [0, q) too, as g1_affine_on_curve
bool g2_on_curve(const g2_affine& p) {
    for (const fe* c : {&p.x.a, &p.x.b, &p.y.a, &p.y.b})
        if (!fe_is_canonical<Fq>(*c)) return false;
    if (p.inf) return true;
    // b' = 3 / (9 + u) = 3 (9 - u) / 82
    const fe inv82 = fe_inv<Fq>(fe_from_u32<Fq>(82));
    const fq2 b = {fe_mul<Fq>(fe_from_u32<Fq>(27), inv82), fe_neg<Fq>(fe_mul<Fq>(fe_from_u32<Fq>(3), inv82))};
    return fq2_eq(fq2_sqr(p.y), fq2_add(fq2_mul(fq2_sqr(p.x), p.x), b));
}

// 128-byte record x0 || x1 || y0 || y1 (Montgomery), the ptau layout read by srs.rs:185-199
g2_affine g2_load(const uint64_t rec[16]) {
    g2_affine p;
    std::memcpy(&p.x.a, rec, 32);
    std::memcpy(&p.x.b, rec + 4, 32);
    std::memcpy(&p.y.a, rec + 8, 32);
    std::memcpy(&p.y.b, rec + 12, 32);
    p.inf = fq2_is_zero(p.x) && fq2_is_zero(p.y);
    return p;
}
g1_affine g1_load(const uint64_t xy[8]) {
    g1_affine p;
    std::memcpy(&p, xy, 64);
    return p;
}

// ---- G1 helpers of the verifier (host XYZZ arithmetic of ec.cuh) -------------------------------------------
// sum_i s_i P_i, collected first and evaluated with ONE chain of doublings (Straus: 254 doublings in all and a mixed
// addition per set scalar bit, instead of 254 doublings per term)
struct G1Sum {
    std::vector<g1_affine> pts;
    std::vector<fe> scalars;  // canonical (non-Montgomery) limbs
    g1_xyzz eval() const {
        g1_xyzz acc = g1_xyzz_inf();
        for (int bit = 253; bit >= 0; --bit) {
            acc = g1_dbl(acc);
            for (size_t i = 0; i < pts.size(); ++i)
                if ((scalars[i].l[bit >> 5] >> (bit & 31)) & 1u) acc = g1_add_mixed(acc, pts[i]);
        }
        return acc;
    }
};
void g1_acc(G1Sum* acc, const g1_affine& p, const fe& s_mont) {
    if (g1_affine_is_inf(p) || fe_is_zero(s_mont)) return;
    acc->pts.push_back(p);
    acc->scalars.push_back(fe_from_mont<Fr>(s_mont));
}
bool pairing_product_is_one(const g1_affine* ps, const g2_affine* qs, size_t k) {
    return fq12_is_one(final_exponentiation(miller_loop_product(ps, qs, k), pairing_consts()));
}

// Host sink of vt::plonk_terms / vt::link_terms: each term goes into the Straus sum of its side
struct HostSink {
    const g1_affine* points;  // indexed by slot
    G1Sum A, B;
    void operator()(int slot, int side, const fe& s) { g1_acc(side == vt::kSideA ? &A : &B, points[slot], s); }
};
// Host denominators of vt::plonk_terms: one inversion per public input, w^j by repeated products
struct HostDen {
    fe zeta, nfr, w, wj;
    size_t next = 0;
    void get(size_t j, fe* inv, fe* wpow) {
        if (j == 0) wj = fe_one<Fr>();
        else if (j == next) wj = fe_mul<Fr>(wj, w);
        next = j + 1;
        *wpow = wj;
        *inv = fe_inv<Fr>(fe_mul<Fr>(fe_sub<Fr>(zeta, wj), nfr));
    }
};

int two_pair_check(const g1_affine& a, const g1_affine& b, const uint64_t g2_tau_h[16], const uint64_t g2_h[16], const char* who,
                   int* accepted) {
    bool one = false;
    const int rc = pairing_two_is_one(a, b, g2_tau_h, g2_h, &one);
    if (rc == B200_ERR_NOT_ON_CURVE) set_error(std::string(who) + ": G2 point not on curve");
    if (rc == B200_OK) *accepted = one ? 1 : 0;
    return rc;
}

}  // namespace

void g2_prepare(const g2_affine& q, G2Prepared* out) {
    g2_affine r = q;
    int step = 0;
    for (int i = 63; i >= 0; --i) {
        out->line[step++] = line_step(&r, r);
        if ((kAteLow >> i) & 1) out->line[step++] = line_step(&r, q);
    }
    const g2_affine q1 = g2_frobenius(q);
    g2_affine nq2 = g2_frobenius(q1);
    nq2.y = fq2_neg(nq2.y);
    out->line[step++] = line_step(&r, q1);
    out->line[step++] = line_step(&r, nq2);
}

bool g2_prepare_record(const uint64_t rec[16], G2Prepared* out) {
    const g2_affine q = g2_load(rec);
    if (!g2_on_curve(q)) return false;
    g2_prepare(q, out);
    return true;
}

bool g2_load_record(const uint64_t rec[16], g2_affine* out) {
    *out = g2_load(rec);
    return g2_on_curve(*out);
}

bool g2_record_on_curve(const uint64_t rec[16]) { return g2_on_curve(g2_load(rec)); }

bool g2_records_on_curve(const uint64_t g2_tau_h[16], const uint64_t g2_h[16]) {
    return g2_on_curve(g2_load(g2_tau_h)) && g2_on_curve(g2_load(g2_h));
}

int pairing_two_is_one(const g1_affine& a, const g1_affine& b, const uint64_t g2_tau_h[16], const uint64_t g2_h[16],
                       bool* is_one) {
    const g1_affine ps[2] = {a, b};
    const g2_affine qs[2] = {g2_load(g2_tau_h), g2_load(g2_h)};
    if (!g2_on_curve(qs[0]) || !g2_on_curve(qs[1])) return B200_ERR_NOT_ON_CURVE;
    *is_one = pairing_product_is_one(ps, qs, 2);
    return B200_OK;
}

}  // namespace b200

using namespace b200;

extern "C" {

int b200_pairing_check(const uint64_t* g1_points, const uint64_t* g2_points, size_t k, int* is_one) {
    B200_TRY
    if ((k && (!g1_points || !g2_points)) || !is_one) return B200_ERR_INVALID;
    std::vector<g1_affine> ps(k);
    std::vector<g2_affine> qs(k);
    for (size_t i = 0; i < k; ++i) {
        ps[i] = g1_load(g1_points + 8 * i);
        qs[i] = g2_load(g2_points + 16 * i);
        if (!g1_affine_on_curve(ps[i]) || !g2_on_curve(qs[i])) {
            set_error("pairing_check: point not on curve");
            return B200_ERR_NOT_ON_CURVE;
        }
    }
    *is_one = pairing_product_is_one(ps.data(), qs.data(), k) ? 1 : 0;
    return B200_OK;
    B200_CATCH
}

int b200_plonk_verify(unsigned log_n, size_t num_inputs, const uint64_t* k, const uint64_t* selector_comms,
                      const uint64_t* sigma_comms, const uint64_t* pub_inputs, const b200_proof* proof_in,
                      const uint64_t g2_h[16], const uint64_t g2_tau_h[16], int* accepted) {
    B200_TRY
    if (!k || !selector_comms || !sigma_comms || !proof_in || !g2_h || !g2_tau_h || !accepted || (num_inputs && !pub_inputs) ||
        log_n > 28)
        return B200_ERR_INVALID;
    *accepted = 0;
    const size_t n = (size_t)1 << log_n;
    const vt::ProofIn& proof = *reinterpret_cast<const vt::ProofIn*>(proof_in);
    const fe* kk = reinterpret_cast<const fe*>(k);
    const g1_affine* sel = reinterpret_cast<const g1_affine*>(selector_comms);
    const g1_affine* sig = reinterpret_cast<const g1_affine*>(sigma_comms);
    const fe* pi = reinterpret_cast<const fe*>(pub_inputs);
    if (!vt::plonk_points_on_curve(sel, sig, proof) || !vt::plonk_scalars_canonical(kk, pi, num_inputs, proof))
        return B200_OK;  // rejected
    // ---- challenges (same transcript as the prover, plonk.cu) ------------------------------------------------
    SolidityTranscript tr;
    const vt::PlonkChallenges ch = vt::plonk_challenges(tr, log_n, num_inputs, kk, sel, sig, pi, proof);
    // ---- A and B (vt::plonk_terms), evaluated on the host ------------------------------------------------------
    HostDen den;
    den.zeta = ch.zeta;
    den.w = host_root_of_unity(log_n);
    den.nfr = fe_zero();
    den.nfr.l[0] = (uint32_t)n;
    den.nfr.l[1] = (uint32_t)((uint64_t)n >> 32);
    den.nfr = fe_to_mont<Fr>(den.nfr);
    g1_affine points[vt::kSlots];
    for (int s = 0; s < vt::kProofPoints; ++s) points[s] = vt::proof_point(proof, s);
    for (int s = 0; s < vt::NS; ++s) points[vt::kSlotSel + s] = sel[s];
    for (int s = 0; s < vt::NW; ++s) points[vt::kSlotSig + s] = sig[s];
    points[vt::kSlotG] = vt::g1_generator();
    HostSink sink{points, {}, {}};
    vt::plonk_terms(log_n, num_inputs, kk, pi, proof, ch, den.w, den, sink);
    // e(A, [tau]_2) == e(B, [1]_2)   <=>   e(A, [tau]_2) * e(-B, [1]_2) == 1
    return two_pair_check(g1_to_affine(sink.A.eval()), g1_affine_neg(g1_to_affine(sink.B.eval())), g2_tau_h, g2_h, "verify",
                          accepted);
    B200_CATCH
}

int b200_plonk_verify_link(const uint64_t* comm1, const uint64_t* comm2, unsigned alignment, size_t offset, size_t size,
                           const b200_link_proof* proof, const uint64_t g2_h[16], const uint64_t g2_tau_h[16], int* accepted) {
    B200_TRY
    // a group of more roots than the 2^alignment-th roots of unity holds has no layout (and Z_D would take `size` products)
    if (!comm1 || !comm2 || !proof || !g2_h || !g2_tau_h || !accepted || alignment > 28 || size == 0 ||
        size > ((size_t)1 << alignment))
        return B200_ERR_INVALID;
    *accepted = 0;
    g1_affine points[vt::kLinkPoints];
    points[vt::kLinkC1] = g1_load(comm1);
    points[vt::kLinkC2] = g1_load(comm2);
    points[vt::kLinkCq] = g1_load(proof->quotient_commitment);
    points[vt::kLinkPi] = g1_load(proof->opening_proof);
    for (const g1_affine& p : points)
        if (!g1_affine_on_curve(p)) return B200_OK;
    SolidityTranscript tr;
    const fe eta = vt::link_challenge(tr, points[vt::kLinkC1], points[vt::kLinkC2], points[vt::kLinkCq]);
    const fe zd = vt::link_zd(eta, host_root_of_unity(alignment), (uint64_t)offset, (uint64_t)size);
    HostSink sink{points, {}, {}};
    vt::link_terms(eta, zd, sink);
    return two_pair_check(g1_to_affine(sink.A.eval()), g1_affine_neg(g1_to_affine(sink.B.eval())), g2_tau_h, g2_h,
                          "verify_link", accepted);
    B200_CATCH
}

}  // extern "C"
