// The verifier's equations, host and device (FF_HD): the ONE definition of how a PlonK proof or a link proof turns
// into the two G1 combinations of its pairing check
//     e(A, [tau]_2) == e(B, [1]_2),
// shared by the single verifiers (verify.cu: host Straus evaluation, then a 2-pair pairing) and the batch verifier
// (verify_batch.cu: one device thread per item, all items merged into one MSM pair and ONE pairing).
//
// A proof is emitted as (slot, A | B, scalar) terms: every slot names one G1 point of the item (its 13 proof
// commitments), of its verifying key (13 selector + 5 sigma commitments) or the generator G.  Each (slot, side) is
// emitted at most once, so a sink can store instead of accumulate.  A link proof uses slots C1, C2, Cq, pi.
#pragma once
#include "b200prover.h"
#include "ec.cuh"
#include "ff.cuh"
#include "transcript.h"

namespace b200 {

namespace vt {

constexpr int NW = 5, NS = 13;

struct ProofIn {  // layout of b200_proof
    g1_affine wires_poly_comms[NW];
    g1_affine prod_perm_poly_comm;
    g1_affine split_quot_poly_comms[NW];
    g1_affine opening_proof;
    g1_affine shifted_opening_proof;
    fe wires_evals[NW];
    fe wire_sigma_evals[NW - 1];
    fe perm_next_eval;
};
static_assert(sizeof(ProofIn) == sizeof(b200_proof), "proof layout");

// slots of a proof item
enum : int {
    kSlotW = 0,     // wires_poly_comms[5]
    kSlotZ = 5,     // prod_perm_poly_comm
    kSlotT = 6,     // split_quot_poly_comms[5]
    kSlotWz = 11,   // opening_proof
    kSlotWzw = 12,  // shifted_opening_proof
    kProofPoints = 13,
    kSlotSel = 13,  // verifying key: selector_comms[13]
    kSlotSig = 26,  // verifying key: sigma_comms[5]
    kVkPoints = 18,
    kSlotG = 31,    // the generator (1, 2)
    kSlots = 32,
};
// slots of a link item
enum : int { kLinkC1 = 0, kLinkC2 = 1, kLinkCq = 2, kLinkPi = 3, kLinkPoints = 4 };
enum : int { kSideA = 0, kSideB = 1 };

FF_HD const g1_affine& proof_point(const ProofIn& p, int slot) {
    if (slot < kSlotZ) return p.wires_poly_comms[slot - kSlotW];
    if (slot == kSlotZ) return p.prod_perm_poly_comm;
    if (slot < kSlotWz) return p.split_quot_poly_comms[slot - kSlotT];
    return slot == kSlotWz ? p.opening_proof : p.shifted_opening_proof;
}

FF_HD g1_affine g1_generator() {
    g1_affine g;
    g.x = fe_one<FqCfg>();
    g.y = fe_from_u32<FqCfg>(2);
    return g;
}

FF_HD fe fr_pow_u64(fe a, uint64_t e) {
    fe r = fe_one<FrCfg>();
    while (e) {
        if (e & 1) r = fe_mul<FrCfg>(r, a);
        a = fe_sqr<FrCfg>(a);
        e >>= 1;
    }
    return r;
}

// every group element the verifier multiplies must be on the curve (the identity is allowed)
FF_HD bool plonk_points_on_curve(const g1_affine* sel, const g1_affine* sig, const ProofIn& proof) {
    bool ok = true;
    for (int i = 0; i < NS; ++i) ok = ok && g1_affine_on_curve(sel[i]);
    for (int i = 0; i < NW; ++i) ok = ok && g1_affine_on_curve(sig[i]);
    for (int s = 0; s < kProofPoints; ++s) ok = ok && g1_affine_on_curve(proof_point(proof, s));
    return ok;
}

// every scalar the verifier reads must be an element of Fr, i.e. below r: the key's k, the public inputs and the
// proof's evaluations.  The transcript reduces what it hashes, so v + r would give the same challenges as v.
FF_HD bool plonk_scalars_canonical(const fe* kk, const fe* pi, size_t num_inputs, const ProofIn& proof) {
    bool ok = true;
    for (int i = 0; i < NW; ++i) ok = ok && fe_is_canonical<FrCfg>(kk[i]);
    for (size_t i = 0; i < num_inputs; ++i) ok = ok && fe_is_canonical<FrCfg>(pi[i]);
    for (int i = 0; i < NW; ++i) ok = ok && fe_is_canonical<FrCfg>(proof.wires_evals[i]);
    for (int i = 0; i < NW - 1; ++i) ok = ok && fe_is_canonical<FrCfg>(proof.wire_sigma_evals[i]);
    return ok && fe_is_canonical<FrCfg>(proof.perm_next_eval);
}

struct PlonkChallenges {
    fe beta, gamma, alpha, zeta, v, u;
};

// the verifier's transcript: the same bytes as the prover's (plonk.cu)
template <class Bytes>
FF_HD PlonkChallenges plonk_challenges(SolidityTranscriptT<Bytes>& tr, unsigned log_n, size_t num_inputs, const fe* kk,
                                       const g1_affine* sel, const g1_affine* sig, const fe* pi, const ProofIn& proof) {
    PlonkChallenges c;
    tr.append_u32_be(254);
    tr.append_u64_be((uint64_t)1 << log_n);
    tr.append_u64_be((uint64_t)num_inputs);
    for (int i = 0; i < NW; ++i) tr.append_field_elem(kk[i]);
    for (int s = 0; s < NS; ++s) tr.append_commitment(sel[s]);
    for (int i = 0; i < NW; ++i) tr.append_commitment(sig[i]);
    for (size_t i = 0; i < num_inputs; ++i) tr.append_field_elem(pi[i]);
    for (int i = 0; i < NW; ++i) tr.append_commitment(proof.wires_poly_comms[i]);
    c.beta = tr.get_and_append_challenge();
    c.gamma = tr.get_and_append_challenge();
    tr.append_commitment(proof.prod_perm_poly_comm);
    c.alpha = tr.get_and_append_challenge();
    for (int i = 0; i < NW; ++i) tr.append_commitment(proof.split_quot_poly_comms[i]);
    c.zeta = tr.get_and_append_challenge();
    for (int i = 0; i < NW; ++i) tr.append_field_elem(proof.wires_evals[i]);
    for (int i = 0; i < NW - 1; ++i) tr.append_field_elem(proof.wire_sigma_evals[i]);
    tr.append_field_elem(proof.perm_next_eval);
    c.v = tr.get_and_append_challenge();
    tr.append_commitment(proof.opening_proof);
    tr.append_commitment(proof.shifted_opening_proof);
    c.u = tr.get_and_append_challenge();
    return c;
}

// Bytes the proof transcript appends (what a device transcript buffer must hold).
FF_HD size_t plonk_transcript_bytes(size_t num_inputs) {
    return 4 + 8 + 8 + 32 * NW + 64 * NS + 64 * NW + 32 * num_inputs + 64 * NW + 64 + 64 * NW + 32 * (2 * NW) + 64 * 2;
}

// The A / B terms of one proof.  `den.get(j, &inv, &wj)` supplies 1 / (n (zeta - w^j)) and w^j for j = 0 (also
// L_1's denominator) and then j = 0 .. num_inputs - 1 in order; w = the domain generator.
//   r0 = PI(zeta) - alpha^2 L1(zeta) - alpha z_w prod_{i<4} (w_i + beta s_i + gamma) (w_4 + gamma)
//   D  = linearisation commitment, F = D + sum v^i [w_i] + sum v^(5+i) [s_i], E = -r0 + sum v^i w_i + ...
//   A  = W_z + u W_zw,   B = zeta W_z + u zeta w W_zw + F - E G + u ([z] - z_w G)
#pragma nv_exec_check_disable
template <class Den, class Sink>
FF_HD void plonk_terms(unsigned log_n, size_t num_inputs, const fe* kk, const fe* pi, const ProofIn& proof,
                       const PlonkChallenges& ch, const fe& w, Den& den, Sink& sink) {
    using Fr = FrCfg;
    const fe one = fe_one<Fr>();
    const fe& beta = ch.beta;
    const fe& gamma = ch.gamma;
    const fe& alpha = ch.alpha;
    const fe& zeta = ch.zeta;
    const fe vanish = fe_sub<Fr>(fr_pow_u64(zeta, (uint64_t)1 << log_n), one);
    fe inv0, w0;
    den.get(0, &inv0, &w0);
    // zeta on the domain makes L_1 / PI denominators vanish: the reference rejects such proofs too (probability ~ n / r)
    const fe l1 = fe_mul<Fr>(vanish, inv0);
    const fe alpha2 = fe_sqr<Fr>(alpha);
    fe pi_eval = fe_zero();
    for (size_t j = 0; j < num_inputs; ++j) {  // PI(zeta) = sum_j pi_j w^j Z_H(zeta) / (n (zeta - w^j))
        fe t, wj;
        den.get(j, &t, &wj);
        t = fe_mul<Fr>(fe_mul<Fr>(fe_mul<Fr>(t, vanish), wj), pi[j]);
        pi_eval = fe_add<Fr>(pi_eval, t);
    }
    const fe* we = proof.wires_evals;
    const fe* se = proof.wire_sigma_evals;
    fe prod = fe_mul<Fr>(alpha, proof.perm_next_eval);
    for (int j = 0; j < NW - 1; ++j) prod = fe_mul<Fr>(prod, fe_add<Fr>(fe_add<Fr>(fe_mul<Fr>(se[j], beta), we[j]), gamma));
    const fe prod4 = fe_mul<Fr>(prod, fe_add<Fr>(we[4], gamma));
    const fe r0 = fe_sub<Fr>(fe_sub<Fr>(pi_eval, fe_mul<Fr>(alpha2, l1)), prod4);

    // ---- D: linearisation commitment ---------------------------------------------------------------------------
    for (int j = 0; j < 4; ++j) sink(kSlotSel + j, kSideB, we[j]);
    sink(kSlotSel + 4, kSideB, fe_mul<Fr>(we[0], we[1]));
    sink(kSlotSel + 5, kSideB, fe_mul<Fr>(we[2], we[3]));
    for (int j = 0; j < 4; ++j) sink(kSlotSel + 6 + j, kSideB, fe_mul<Fr>(fe_sqr<Fr>(fe_sqr<Fr>(we[j])), we[j]));
    sink(kSlotSel + 10, kSideB, fe_neg<Fr>(we[4]));
    sink(kSlotSel + 11, kSideB, one);
    sink(kSlotSel + 12, kSideB, fe_mul<Fr>(fe_mul<Fr>(fe_mul<Fr>(we[0], we[1]), fe_mul<Fr>(we[2], we[3])), we[4]));
    fe coeff = alpha;
    for (int j = 0; j < NW; ++j)
        coeff = fe_mul<Fr>(coeff, fe_add<Fr>(fe_add<Fr>(fe_mul<Fr>(fe_mul<Fr>(kk[j], zeta), beta), we[j]), gamma));
    coeff = fe_add<Fr>(coeff, fe_mul<Fr>(alpha2, l1));
    sink(kSlotZ, kSideB, fe_add<Fr>(coeff, ch.u));  // D's term plus the u [z] of B
    sink(kSlotSig + NW - 1, kSideB, fe_neg<Fr>(fe_mul<Fr>(prod, beta)));
    const fe zn2 = fe_mul<Fr>(fe_mul<Fr>(fe_add<Fr>(vanish, one), zeta), zeta);
    fe c = fe_neg<Fr>(vanish);
    for (int i = 0; i < NW; ++i) {
        sink(kSlotT + i, kSideB, c);
        c = fe_mul<Fr>(c, zn2);
    }
    // ---- F, E: batched opening at zeta -------------------------------------------------------------------------
    fe E = fe_neg<Fr>(r0), vp = one;
    for (int i = 0; i < NW; ++i) {
        vp = fe_mul<Fr>(vp, ch.v);
        sink(kSlotW + i, kSideB, vp);
        E = fe_add<Fr>(E, fe_mul<Fr>(vp, we[i]));
    }
    for (int i = 0; i < NW - 1; ++i) {
        vp = fe_mul<Fr>(vp, ch.v);
        sink(kSlotSig + i, kSideB, vp);
        E = fe_add<Fr>(E, fe_mul<Fr>(vp, se[i]));
    }
    // ---- pairing operands ----------------------------------------------------------------------------------------
    sink(kSlotG, kSideB, fe_neg<Fr>(fe_add<Fr>(E, fe_mul<Fr>(ch.u, proof.perm_next_eval))));
    sink(kSlotWz, kSideA, one);
    sink(kSlotWz, kSideB, zeta);
    sink(kSlotWzw, kSideA, ch.u);
    sink(kSlotWzw, kSideB, fe_mul<Fr>(ch.u, fe_mul<Fr>(zeta, w)));
}

// ---- link proofs ---------------------------------------------------------------------------------------------
template <class Bytes>
FF_HD fe link_challenge(SolidityTranscriptT<Bytes>& tr, const g1_affine& c1, const g1_affine& c2, const g1_affine& cq) {
    tr.append_commitment(c1);
    tr.append_commitment(c2);
    tr.append_commitment(cq);
    return tr.get_and_append_challenge();
}
constexpr size_t kLinkTranscriptBytes = 3 * 64;

// Z_D(eta) = prod_{i < size} (eta - g^(offset + i)), serially
FF_HD fe link_zd(const fe& eta, const fe& g, uint64_t offset, uint64_t size) {
    fe root = fr_pow_u64(g, offset), zd = fe_one<FrCfg>();
    for (uint64_t i = 0; i < size; ++i) {
        zd = fe_mul<FrCfg>(zd, fe_sub<FrCfg>(eta, root));
        root = fe_mul<FrCfg>(root, g);
    }
    return zd;
}

// (tau - eta) pi == C1 - C2 - Z_D(eta) Cq   <=>   e(pi, [tau]_2) == e(C1 - C2 - Z_D(eta) Cq + eta pi, [1]_2)
#pragma nv_exec_check_disable
template <class Sink>
FF_HD void link_terms(const fe& eta, const fe& zd, Sink& sink) {
    const fe one = fe_one<FrCfg>();
    sink(kLinkC1, kSideB, one);
    sink(kLinkC2, kSideB, fe_neg<FrCfg>(one));
    sink(kLinkCq, kSideB, fe_neg<FrCfg>(zd));
    sink(kLinkPi, kSideA, one);
    sink(kLinkPi, kSideB, eta);
}

}  // namespace vt

// ---- host pairing of verify.cu, for the batch verifier --------------------------------------------------------
// e(a, g2_tau_h) * e(b, g2_h) == 1.  B200_ERR_NOT_ON_CURVE when a G2 record is off the curve.
int pairing_two_is_one(const g1_affine& a, const g1_affine& b, const uint64_t g2_tau_h[16], const uint64_t g2_h[16],
                       bool* is_one);
bool g2_records_on_curve(const uint64_t g2_tau_h[16], const uint64_t g2_h[16]);

}  // namespace b200
