// Batch verification of PlonK proofs and link proofs: every item's check has the form e(A_i, [tau]_2) == e(B_i, [1]_2)
// with A_i, B_i linear combinations of known G1 points (verify_terms.h), so with random weights rho_i the k checks
// collapse into ONE pairing check
//     e(sum rho_i A_i, [tau]_2) == e(sum rho_i B_i, [1]_2),
// i.e. two MSMs over the batch's points (one msm_device_batch call, batch = 2) and one 2-pair pairing on the host.
//
// Pipeline (one device thread per item where the work is per item):
//   1. k_prepare: on-curve check of the item's G1 points, its SolidityTranscript (transcript.h, in a per-item slice of
//      device memory sized for it), the challenges, the item digest, and for a proof its denominators
//      n (zeta - w^j), j < max(1, num_inputs) (j = 0 is also L_1's); for a link Z_D(eta), serially.
//   2. batch_inverse_enqueue over all denominators (plonk.cu).
//   3. Randomisers by Fiat–Shamir over the whole batch, so a prover cannot predict them:
//        d_i  = keccak(tag_i || final transcript state_i || what that transcript did not absorb)
//               tag 0 for a proof (nothing left out), tag 1 for a link (its opening pi and its layout
//               alignment u32 || offset u64 || size u64, big-endian, in the transcript's encoding);
//        seed = keccak("b200 batch verify v1" || d_0 || ... || d_{k-1} || g2_h || g2_tau_h)   (host, k x 32 bytes);
//        rho_i = keccak(seed || i as u64 big-endian), read as a big-endian integer mod r (1 if that is 0).
//   4. k_scalars: rho_i times every A / B coefficient of the item (vt::plonk_terms / vt::link_terms).
//   5. k_merge_items / k_merge_shared: the MSM scalar vectors under a mask of items.  The items' own points keep their
//      scalars; the 18 verifying-key points are summed per distinct key over its items and G over all items (a segmented
//      reduction), so a batch of one circuit has ~13 bases per proof plus 19 shared ones.  Identity bases get scalar 0.
//   6. Bases (gathered on the device by k_gather_bases, no window tables: they are used once), msm_device_batch with
//      A and B, and ONE pairing.  If it fails and verdicts are asked for, the failing items are found by bisection:
//      each step re-merges a subset from the per-item scalars already on the device (masked merge, MSM, one pairing).
// An item with an off-curve point or a field element outside [0, p) is rejected and left out of the combination.
#include <cstring>
#include <mutex>
#include <vector>

#include "b200prover.h"
#include "device_ctx.h"
#include "transcript.h"
#include "verify_terms.h"

namespace b200 {

namespace {

using Fr = FrCfg;
constexpr int kMaxAlign = 28;

struct VkDev {  // one distinct verifying key
    fe k[vt::NW];
    g1_affine sel[vt::NS], sig[vt::NW];
    fe w;      // domain generator
    fe n_mont; // n in Montgomery form
    uint64_t num_inputs;
    uint64_t wtab_off;  // w^j, j < max(1, num_inputs), at wtab + wtab_off
    uint32_t log_n;
};
struct LinkDev {
    g1_affine pt[vt::kLinkPoints];  // C1, C2, Cq, pi
    uint64_t offset, size;
    uint32_t alignment;
};
struct ItemDev {
    uint32_t kind;  // 0 proof, 1 link
    uint32_t idx;   // into the proofs or the links
    uint32_t vk;
    uint32_t base_off;  // first of its own bases
    uint64_t pi_off, den_off, tr_off, tr_cap;
};
struct ItemState {  // what k_prepare leaves for k_scalars
    vt::PlonkChallenges ch;  // link: zeta = eta, beta = Z_D(eta)
    uint32_t ok;             // every point on the curve, every scalar below r (and the transcript fitted its buffer)
};
struct Roots {
    fe g[kMaxAlign + 1];  // generator of the 2^a-th roots of unity
};
struct Seed {
    uint8_t b[32];
};

// record of one item's scaled coefficients: [side][slot]
constexpr int kRec = 2 * vt::kSlots;

struct DevDen {  // vt::plonk_terms denominators from the batch-inverted table
    const fe* inv;
    const fe* wpow;
    FF_D void get(size_t j, fe* i, fe* w) const {
        *i = fe_load(inv + j);
        *w = fe_load(wpow + j);
    }
};
struct DevSink {
    fe* rec;
    fe rho;
    FF_D void operator()(int slot, int side, const fe& s) const { fe_store(rec + side * vt::kSlots + slot, fe_mul<Fr>(rho, s)); }
};

__global__ void __launch_bounds__(128) k_prepare(const ItemDev* __restrict__ items, size_t k, const VkDev* __restrict__ vks,
                                                 const vt::ProofIn* __restrict__ proofs, const LinkDev* __restrict__ links,
                                                 const fe* __restrict__ pi, const fe* __restrict__ wtab, uint8_t* tr_bytes,
                                                 fe* __restrict__ den, Roots roots, ItemState* __restrict__ st,
                                                 uint8_t* __restrict__ digest) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= k) return;
    const ItemDev it = items[i];
    ItemState out;
    Keccak256 dg;
    if (it.kind == 0) {
        const VkDev& vk = vks[it.vk];
        const vt::ProofIn& proof = proofs[it.idx];
        bool ok = vt::plonk_points_on_curve(vk.sel, vk.sig, proof) &&
                  vt::plonk_scalars_canonical(vk.k, pi + it.pi_off, vk.num_inputs, proof);
        SolidityTranscriptT<SpanBytes> tr(SpanBytes{tr_bytes + it.tr_off, 0, it.tr_cap, false});
        out.ch = vt::plonk_challenges(tr, vk.log_n, vk.num_inputs, vk.k, vk.sel, vk.sig, pi + it.pi_off, proof);
        ok = ok && !tr.bytes().overflow;
        out.ok = ok;
        const uint64_t nd = vk.num_inputs ? vk.num_inputs : 1;
        for (uint64_t j = 0; j < nd; ++j)
            fe_store(den + it.den_off + j, fe_mul<Fr>(fe_sub<Fr>(out.ch.zeta, fe_load(wtab + vk.wtab_off + j)), vk.n_mont));
        dg.absorb_byte(0);
        dg.absorb(tr.state(), 64);
    } else {
        const LinkDev& l = links[it.idx];
        bool ok = true;
        for (int p = 0; p < vt::kLinkPoints; ++p) ok = ok && g1_affine_on_curve(l.pt[p]);
        uint8_t buf[vt::kLinkTranscriptBytes];
        SolidityTranscriptT<SpanBytes> tr(SpanBytes{buf, 0, sizeof(buf), false});
        const fe eta = vt::link_challenge(tr, l.pt[vt::kLinkC1], l.pt[vt::kLinkC2], l.pt[vt::kLinkCq]);
        out.ch.zeta = eta;
        out.ch.beta = ok ? vt::link_zd(eta, roots.g[l.alignment], l.offset, l.size) : fe_zero();
        out.ok = ok && !tr.bytes().overflow;
        // the link's digest also binds what its transcript left out: pi and the layout
        uint8_t rest[64 + 4 + 8 + 8];
        SolidityTranscriptT<SpanBytes> extra(SpanBytes{rest, 0, sizeof(rest), false});
        extra.append_commitment(l.pt[vt::kLinkPi]);
        extra.append_u32_be(l.alignment);
        extra.append_u64_be(l.offset);
        extra.append_u64_be(l.size);
        dg.absorb_byte(1);
        dg.absorb(tr.state(), 64);
        dg.absorb(rest, sizeof(rest));
    }
    st[i] = out;
    uint8_t d[32];
    dg.finish(d);
    for (int b = 0; b < 32; ++b) digest[32 * i + b] = d[b];
}

__global__ void __launch_bounds__(128) k_scalars(const ItemDev* __restrict__ items, size_t k, const VkDev* __restrict__ vks,
                                                 const vt::ProofIn* __restrict__ proofs, const fe* __restrict__ pi,
                                                 const fe* __restrict__ wtab, const fe* __restrict__ den_inv,
                                                 const ItemState* __restrict__ st, Seed seed, fe* __restrict__ rec) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= k) return;
    const ItemState s = st[i];
    if (!s.ok) return;  // rejected: its record stays zero
    // rho_i = keccak(seed || i) mod r
    uint8_t h[32];
    {
        Keccak256 kc;
        kc.absorb(seed.b, 32);
        uint8_t be[8];
        for (int b = 0; b < 8; ++b) be[b] = (uint8_t)((uint64_t)i >> (56 - 8 * b));
        kc.absorb(be, 8);
        kc.finish(h);
    }
    fe rho = fe_zero();
    const fe c256 = fe_from_u32<Fr>(256);
    for (int b = 0; b < 32; ++b) rho = fe_add<Fr>(fe_mul<Fr>(rho, c256), fe_from_u32<Fr>(h[b]));
    if (fe_is_zero(rho)) rho = fe_one<Fr>();
    const ItemDev it = items[i];
    DevSink sink{rec + i * kRec, rho};
    if (it.kind == 0) {
        const VkDev& vk = vks[it.vk];
        DevDen dd{den_inv + it.den_off, wtab + vk.wtab_off};
        vt::plonk_terms(vk.log_n, vk.num_inputs, vk.k, pi + it.pi_off, proofs[it.idx], s.ch, vk.w, dd, sink);
    } else {
        vt::link_terms(s.ch.zeta, s.ch.beta, sink);
    }
}

// the items' own points, in base order
__global__ void k_gather_bases(const ItemDev* __restrict__ items, size_t k, const vt::ProofIn* __restrict__ proofs,
                               const LinkDev* __restrict__ links, g1_affine* __restrict__ bases) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= k) return;
    const ItemDev it = items[i];
    if (it.kind == 0)
        for (int s = 0; s < vt::kProofPoints; ++s) bases[it.base_off + s] = vt::proof_point(proofs[it.idx], s);
    else
        for (int s = 0; s < vt::kLinkPoints; ++s) bases[it.base_off + s] = links[it.idx].pt[s];
}

// scalars of the items' own bases: A at scal[b], B at scal[n_bases + b]; items outside the mask get 0
__global__ void k_merge_items(const ItemDev* __restrict__ items, size_t k, const uint8_t* __restrict__ mask,
                              const fe* __restrict__ rec, const g1_affine* __restrict__ bases, size_t n_bases,
                              fe* __restrict__ scal) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= k) return;
    const ItemDev it = items[i];
    const int np = it.kind == 0 ? vt::kProofPoints : vt::kLinkPoints;
    const bool on = mask[i];
    for (int s = 0; s < np; ++s) {
        const size_t b = it.base_off + s;
        const bool use = on && !g1_affine_is_inf(bases[b]);
        fe_store(scal + b, use ? fe_load(rec + i * kRec + s) : fe_zero());
        fe_store(scal + n_bases + b, use ? fe_load(rec + i * kRec + vt::kSlots + s) : fe_zero());
    }
}

// Shared bases: block v * 18 + s sums slot kSlotSel + s of the items of key v (CSR list), the last block sums G over
// all items.  A strided sum per thread, then a shared-memory tree.
constexpr int kMergeThreads = 128;
__global__ void __launch_bounds__(kMergeThreads) k_merge_shared(const uint32_t* __restrict__ vk_items,
                                                                const uint32_t* __restrict__ vk_start, unsigned n_vks, size_t k,
                                                                const uint8_t* __restrict__ mask, const fe* __restrict__ rec,
                                                                const g1_affine* __restrict__ bases, size_t shared0,
                                                                size_t n_bases, fe* __restrict__ scal) {
    __shared__ fe part[kMergeThreads];
    const unsigned blk = blockIdx.x;
    const bool is_g = blk == n_vks * vt::kVkPoints;
    const int slot = is_g ? vt::kSlotG : vt::kSlotSel + (int)(blk % vt::kVkPoints);
    const size_t beg = is_g ? 0 : vk_start[blk / vt::kVkPoints], end = is_g ? k : vk_start[blk / vt::kVkPoints + 1];
    fe acc = fe_zero();
    for (size_t j = beg + threadIdx.x; j < end; j += kMergeThreads) {
        const size_t i = is_g ? j : vk_items[j];
        if (mask[i]) acc = fe_add<Fr>(acc, fe_load(rec + i * kRec + vt::kSlots + slot));
    }
    part[threadIdx.x] = acc;
    __syncthreads();
    for (unsigned off = kMergeThreads / 2; off; off >>= 1) {
        if (threadIdx.x < off) part[threadIdx.x] = fe_add<Fr>(part[threadIdx.x], part[threadIdx.x + off]);
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        const size_t b = shared0 + blk;
        fe_store(scal + b, fe_zero());
        fe_store(scal + n_bases + b, g1_affine_is_inf(bases[b]) ? fe_zero() : part[0]);
    }
}

inline unsigned grid_of(size_t n, unsigned bs) { return (unsigned)((n + bs - 1) / bs); }

template <class T>
int upload(DevBuf* d, const std::vector<T>& h, cudaStream_t st) {
    int rc = d->reserve(h.size() * sizeof(T) + 32);
    if (rc != B200_OK) return rc;
    if (!h.empty()) B200_CUDA(cudaMemcpyAsync(d->p, h.data(), h.size() * sizeof(T), cudaMemcpyHostToDevice, st));
    return B200_OK;
}

struct Batch {
    Context* c;
    size_t k = 0, n_bases = 0, shared0 = 0;
    unsigned n_vks = 0;
    DevBuf items, vks, proofs, links, pi, wtab, tr, den, den_tmp, state, digest, rec, bases_pts, scal, mask, vk_items, vk_start;
    Bases* bases = nullptr;
    ~Batch() { delete bases; }

    // the combined check over the items with mask[i] = 1
    int check(const std::vector<uint8_t>& mask, const uint64_t g2_tau_h[16], const uint64_t g2_h[16], bool* ok) {
        cudaStream_t st = c->stream;
        B200_CUDA(cudaMemcpyAsync(this->mask.p, mask.data(), k, cudaMemcpyHostToDevice, st));
        B200_LAUNCH(k_merge_items, grid_of(k, 128), 128, 0, st)((const ItemDev*)items.p, k, (const uint8_t*)this->mask.p,
                                                               (const fe*)rec.p, (const g1_affine*)bases_pts.p, n_bases,
                                                               (fe*)scal.p);
        B200_LAUNCH(k_merge_shared, n_vks * vt::kVkPoints + 1, kMergeThreads, 0, st)(
            (const uint32_t*)vk_items.p, (const uint32_t*)vk_start.p, n_vks, k, (const uint8_t*)this->mask.p, (const fe*)rec.p,
            (const g1_affine*)bases_pts.p, shared0, n_bases, (fe*)scal.p);
        B200_CUDA(cudaGetLastError());
        g1_affine out[2];
        int inf[2];
        int rc = msm_device_batch(bases, 0, (const fe*)scal.p, n_bases, n_bases, 2, 1, &c->msm, st, out, inf);
        if (rc != B200_OK) return rc;
        for (int j = 0; j < 2; ++j)
            if (inf[j]) out[j].x = out[j].y = fe_zero();
        return pairing_two_is_one(out[0], g1_affine_neg(out[1]), g2_tau_h, g2_h, ok);
    }

    // verdicts of the items listed in `idx` (all valid), whose combined check is known to fail
    int bisect(const std::vector<uint32_t>& idx, const uint64_t g2_tau_h[16], const uint64_t g2_h[16], uint8_t* verdicts) {
        if (idx.size() == 1) {
            verdicts[idx[0]] = 0;
            return B200_OK;
        }
        const std::vector<uint32_t> lo(idx.begin(), idx.begin() + idx.size() / 2), hi(idx.begin() + idx.size() / 2, idx.end());
        std::vector<uint8_t> m(k, 0);
        for (uint32_t i : lo) m[i] = 1;
        bool lo_ok = false;
        int rc = check(m, g2_tau_h, g2_h, &lo_ok);
        if (rc != B200_OK) return rc;
        if (!lo_ok) {
            if ((rc = bisect(lo, g2_tau_h, g2_h, verdicts)) != B200_OK) return rc;
            std::fill(m.begin(), m.end(), 0);
            for (uint32_t i : hi) m[i] = 1;
            bool hi_ok = false;
            if ((rc = check(m, g2_tau_h, g2_h, &hi_ok)) != B200_OK) return rc;
            return hi_ok ? B200_OK : bisect(hi, g2_tau_h, g2_h, verdicts);
        }
        // the whole set fails and its lower half passes: the upper half fails (the check is a product over the items)
        return bisect(hi, g2_tau_h, g2_h, verdicts);
    }
};

}  // namespace

}  // namespace b200

using namespace b200;

extern "C" int b200_plonk_batch_verify(b200_ctx* ctx, const b200_verifying_key* vks, size_t n_vks, const b200_batch_proof* proofs,
                                       size_t n_proofs, const b200_batch_link* links, size_t n_links, const uint64_t g2_h[16],
                                       const uint64_t g2_tau_h[16], int* all_accepted, uint8_t* verdicts) {
    B200_TRY
    if (!ctx || (n_vks && !vks) || (n_proofs && !proofs) || (n_links && !links) || !g2_h || !g2_tau_h || !all_accepted ||
        n_vks > 0xffffffffu || n_proofs + n_links > 0xffffffffu)
        return B200_ERR_INVALID;
    *all_accepted = 0;
    for (size_t v = 0; v < n_vks; ++v)
        if (vks[v].log_n > kMaxAlign || !vks[v].k || !vks[v].selector_comms || !vks[v].sigma_comms) {
            set_error("batch_verify: bad verifying key");
            return B200_ERR_INVALID;
        }
    for (size_t p = 0; p < n_proofs; ++p)
        if (proofs[p].vk >= n_vks || !proofs[p].proof || (vks[proofs[p].vk].num_inputs && !proofs[p].pub_inputs)) {
            set_error("batch_verify: bad proof entry (vk index, proof or public inputs)");
            return B200_ERR_INVALID;
        }
    for (size_t l = 0; l < n_links; ++l)
        if (!links[l].comm1 || !links[l].comm2 || !links[l].proof || links[l].alignment > kMaxAlign || links[l].size == 0) {
            set_error("batch_verify: bad link entry");
            return B200_ERR_INVALID;
        }
    if (!g2_records_on_curve(g2_tau_h, g2_h)) {
        set_error("batch_verify: G2 point not on curve");
        return B200_ERR_NOT_ON_CURVE;
    }
    const size_t k = n_proofs + n_links;
    if (k == 0) {
        *all_accepted = 1;
        return B200_OK;
    }
    std::lock_guard<std::mutex> lk(ctx->c.mu);
    B200_CUDA(cudaSetDevice(ctx->c.device));
    cudaStream_t st = ctx->c.stream;
    Batch bt;
    bt.c = &ctx->c;
    bt.k = k;
    bt.n_vks = (unsigned)n_vks;

    // ---- host staging: keys, items, public inputs, layouts ---------------------------------------------------------
    std::vector<VkDev> hv(n_vks);
    std::vector<fe> hw;  // per key: w and the table start
    size_t wtab_n = 0;
    for (size_t v = 0; v < n_vks; ++v) {
        VkDev& d = hv[v];
        std::memcpy(d.k, vks[v].k, sizeof(d.k));
        std::memcpy(d.sel, vks[v].selector_comms, sizeof(d.sel));
        std::memcpy(d.sig, vks[v].sigma_comms, sizeof(d.sig));
        d.log_n = vks[v].log_n;
        d.num_inputs = vks[v].num_inputs;
        d.w = host_root_of_unity(d.log_n);
        const uint64_t n = (uint64_t)1 << d.log_n;
        fe nf = fe_zero();
        nf.l[0] = (uint32_t)n;
        nf.l[1] = (uint32_t)(n >> 32);
        d.n_mont = fe_to_mont<Fr>(nf);
        d.wtab_off = wtab_n;
        wtab_n += d.num_inputs ? d.num_inputs : 1;
    }
    std::vector<ItemDev> hi(k);
    std::vector<vt::ProofIn> hp(n_proofs);
    std::vector<LinkDev> hl(n_links);
    std::vector<fe> hpi;
    size_t den_n = 0, tr_n = 0, base_n = 0;
    std::vector<std::vector<uint32_t>> per_vk(n_vks);
    for (size_t p = 0; p < n_proofs; ++p) {
        const VkDev& vk = hv[proofs[p].vk];
        std::memcpy(&hp[p], proofs[p].proof, sizeof(vt::ProofIn));
        ItemDev& it = hi[p];
        it.kind = 0;
        it.idx = (uint32_t)p;
        it.vk = proofs[p].vk;
        it.base_off = (uint32_t)base_n;
        base_n += vt::kProofPoints;
        it.pi_off = hpi.size();
        const fe* pi = reinterpret_cast<const fe*>(proofs[p].pub_inputs);
        hpi.insert(hpi.end(), pi, pi + vk.num_inputs);
        it.den_off = den_n;
        den_n += vk.num_inputs ? vk.num_inputs : 1;
        it.tr_off = tr_n;
        it.tr_cap = vt::plonk_transcript_bytes(vk.num_inputs);
        tr_n += it.tr_cap;
        per_vk[it.vk].push_back((uint32_t)p);
    }
    for (size_t l = 0; l < n_links; ++l) {
        LinkDev& d = hl[l];
        std::memcpy(&d.pt[vt::kLinkC1], links[l].comm1, 64);
        std::memcpy(&d.pt[vt::kLinkC2], links[l].comm2, 64);
        std::memcpy(&d.pt[vt::kLinkCq], links[l].proof->quotient_commitment, 64);
        std::memcpy(&d.pt[vt::kLinkPi], links[l].proof->opening_proof, 64);
        d.offset = links[l].offset;
        d.size = links[l].size;
        d.alignment = links[l].alignment;
        ItemDev& it = hi[n_proofs + l];
        std::memset(&it, 0, sizeof(it));
        it.kind = 1;
        it.idx = (uint32_t)l;
        it.base_off = (uint32_t)base_n;
        base_n += vt::kLinkPoints;
    }
    // shared bases after the items' own: 18 per key, then G
    bt.shared0 = base_n;
    bt.n_bases = base_n + n_vks * vt::kVkPoints + 1;
    if (bt.n_bases > 0xffffffffu) return B200_ERR_INVALID;
    std::vector<g1_affine> hshared;
    for (size_t v = 0; v < n_vks; ++v) {
        hshared.insert(hshared.end(), hv[v].sel, hv[v].sel + vt::NS);
        hshared.insert(hshared.end(), hv[v].sig, hv[v].sig + vt::NW);
    }
    hshared.push_back(vt::g1_generator());
    std::vector<uint32_t> hvk_items, hvk_start(n_vks + 1, 0);
    for (size_t v = 0; v < n_vks; ++v) {
        hvk_start[v] = (uint32_t)hvk_items.size();
        hvk_items.insert(hvk_items.end(), per_vk[v].begin(), per_vk[v].end());
    }
    hvk_start[n_vks] = (uint32_t)hvk_items.size();
    Roots roots;
    for (int a = 0; a <= kMaxAlign; ++a) roots.g[a] = host_root_of_unity((unsigned)a);

    int rc;
    if ((rc = upload(&bt.items, hi, st)) || (rc = upload(&bt.vks, hv, st)) || (rc = upload(&bt.proofs, hp, st)) ||
        (rc = upload(&bt.links, hl, st)) || (rc = upload(&bt.pi, hpi, st)) || (rc = upload(&bt.vk_items, hvk_items, st)) ||
        (rc = upload(&bt.vk_start, hvk_start, st)) || (rc = bt.wtab.reserve(wtab_n * sizeof(fe))) ||
        (rc = bt.tr.reserve(tr_n + 1)) || (rc = bt.den.reserve(den_n * sizeof(fe) + 32)) ||
        (rc = bt.den_tmp.reserve(den_n * sizeof(fe) + 32)) || (rc = bt.state.reserve(k * sizeof(ItemState))) ||
        (rc = bt.digest.reserve(k * 32)) || (rc = bt.rec.reserve(k * kRec * sizeof(fe))) ||
        (rc = bt.bases_pts.reserve(bt.n_bases * sizeof(g1_affine))) || (rc = bt.scal.reserve(2 * bt.n_bases * sizeof(fe))) ||
        (rc = bt.mask.reserve(k)))
        return rc;
    // w^j tables of the keys
    for (size_t v = 0; v < n_vks; ++v)
        fill_powers((fe*)bt.wtab.p + hv[v].wtab_off, hv[v].num_inputs ? hv[v].num_inputs : 1, hv[v].w, fe_one<Fr>(), st);
    B200_CUDA(cudaMemcpyAsync((g1_affine*)bt.bases_pts.p + bt.shared0, hshared.data(), hshared.size() * sizeof(g1_affine),
                              cudaMemcpyHostToDevice, st));
    B200_CUDA(cudaMemsetAsync(bt.rec.p, 0, k * kRec * sizeof(fe), st));

    // ---- 1. prepare, 2. invert ------------------------------------------------------------------------------------
    B200_LAUNCH(k_prepare, grid_of(k, 128), 128, 0, st)((const ItemDev*)bt.items.p, k, (const VkDev*)bt.vks.p,
                                                       (const vt::ProofIn*)bt.proofs.p, (const LinkDev*)bt.links.p,
                                                       (const fe*)bt.pi.p, (const fe*)bt.wtab.p, (uint8_t*)bt.tr.p,
                                                       (fe*)bt.den.p, roots, (ItemState*)bt.state.p, (uint8_t*)bt.digest.p);
    if (den_n) batch_inverse_enqueue(nullptr, (fe*)bt.den.p, (fe*)bt.den_tmp.p, den_n, st);
    B200_LAUNCH(k_gather_bases, grid_of(k, 128), 128, 0, st)((const ItemDev*)bt.items.p, k, (const vt::ProofIn*)bt.proofs.p,
                                                            (const LinkDev*)bt.links.p, (g1_affine*)bt.bases_pts.p);
    B200_CUDA(cudaGetLastError());
    // ---- 3. randomisers: seed over all the item digests --------------------------------------------------------------
    std::vector<uint8_t> hdig(k * 32);
    std::vector<ItemState> hst(k);
    B200_CUDA(cudaMemcpyAsync(hdig.data(), bt.digest.p, k * 32, cudaMemcpyDeviceToHost, st));
    B200_CUDA(cudaMemcpyAsync(hst.data(), bt.state.p, k * sizeof(ItemState), cudaMemcpyDeviceToHost, st));
    B200_CUDA(cudaStreamSynchronize(st));
    Seed seed;
    {
        static const char tag[] = "b200 batch verify v1";
        Keccak256 kc;
        kc.absorb(reinterpret_cast<const uint8_t*>(tag), sizeof(tag) - 1);
        kc.absorb(hdig.data(), hdig.size());
        kc.absorb(reinterpret_cast<const uint8_t*>(g2_h), 128);
        kc.absorb(reinterpret_cast<const uint8_t*>(g2_tau_h), 128);
        kc.finish(seed.b);
    }
    // ---- 4. scaled coefficients --------------------------------------------------------------------------------------
    B200_LAUNCH(k_scalars, grid_of(k, 128), 128, 0, st)((const ItemDev*)bt.items.p, k, (const VkDev*)bt.vks.p,
                                                       (const vt::ProofIn*)bt.proofs.p, (const fe*)bt.pi.p,
                                                       (const fe*)bt.wtab.p, (const fe*)bt.den.p,
                                                       (const ItemState*)bt.state.p, seed, (fe*)bt.rec.p);
    B200_CUDA(cudaGetLastError());
    // ---- 5, 6. bases without tables, merged scalars, MSM pair, one pairing ------------------------------------------
    if ((rc = bases_create_device((const g1_affine*)bt.bases_pts.p, bt.n_bases, 1, st, &bt.bases, 0)) != B200_OK) return rc;
    std::vector<uint8_t> mask(k);
    std::vector<uint32_t> valid;
    for (size_t i = 0; i < k; ++i) {
        mask[i] = hst[i].ok ? 1 : 0;
        if (mask[i]) valid.push_back((uint32_t)i);
    }
    bool ok = true;
    if (!valid.empty() && (rc = bt.check(mask, g2_tau_h, g2_h, &ok)) != B200_OK) return rc;
    *all_accepted = ok && valid.size() == k ? 1 : 0;
    if (verdicts) {
        for (size_t i = 0; i < k; ++i) verdicts[i] = mask[i];
        if (!ok && (rc = bt.bisect(valid, g2_tau_h, g2_h, verdicts)) != B200_OK) return rc;
    }
    return B200_OK;
    B200_CATCH
}
