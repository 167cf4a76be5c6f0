// TurboPlonk / KZG prover rounds on the device.
//
// Replaces what the reference calls at
//   /root/reference/crates/circuits/circuit-types/src/traits.rs:850
//       PlonkKzgSnark::<Bn254>::preprocess(&SYSTEM_SRS, &cs)            -> b200_plonk_preprocess
//   /root/reference/crates/circuits/circuit-types/src/traits.rs:996
//       PlonkKzgSnark::prove_with_link_hint::<_, _, SolidityTranscript> -> b200_plonk_prove
// (the algorithm is mpc-jellyfish's TurboPlonk prover, restated in SURVEY.md App. A: 5 wire
// columns, 13 selectors, quotient over the 8n coset, 5-way split, Keccak transcript).
//
// Device-first layout: everything a proof needs that does not depend on the witness is resident in
// HBM per proving key — selector/sigma coefficients, sigma evaluations, and the 18 coset
// evaluation vectors over the 8n domain (302 MB at n = 2^16; the 80 GB of an H100 hold over two hundred
// keys) — so a proof runs 7 size-8n coset NTTs instead of the reference's 25.  Polynomials never
// leave the device between rounds; the host sees 13 commitments and 10 evaluations and runs the
// (serial, few-KB) Keccak transcript between rounds.
#include <algorithm>
#include <chrono>
#include <cstring>
#include <vector>

#include "b200prover.h"
#include "b200settlement.h"
#include "device_ctx.h"
#include "transcript.h"
#include "verify_terms.h"

namespace b200 {

namespace {

constexpr int NW = 5;    // wire columns (GATE_WIDTH + 1)
constexpr int NS = 13;   // q_lc[4] q_mul[2] q_hash[4] q_o q_c q_ecc
constexpr int CH = 16;   // elements per thread in the chunked scans: every level is a chain of CH dependent products
                         // (latency-bound kernels), so short chunks and one more level beat long chunks

struct KArr {
    fe v[NW];
};

using Fr = FrCfg;
#define FMUL(a, b) fe_mul<Fr>((a), (b))
#define FADD(a, b) fe_add<Fr>((a), (b))
#define FSUB(a, b) fe_sub<Fr>((a), (b))

// ---- key setup ---------------------------------------------------------------------------------
// sigma_i(w^j) = k_{i'} * w^{j'} where (i', j') is the image of wire position (i, j)
__global__ void k_sigma_evals(const uint64_t* __restrict__ perm, const fe* __restrict__ dom, size_t n, KArr k,
                              fe* __restrict__ out) {
    const size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= NW * n) return;
    const uint64_t tgt = perm[t];
    fe_store(out + t, FMUL(k.v[tgt / n], fe_load_ro(dom + tgt % n)));
}

// ---- wire table from the witness vector ------------------------------------------------------------
// wires_ev[p][t] = witness_p[wire_vars[t]] for every wire position t = i*n + j of every proof p of a chunk (blockIdx.y), and
// the public inputs — the values on the output wire of rows 0..num_inputs-1 — into the head of pi_poly[p].  The index
// loads and the stores are coalesced; the 32-byte elements come through the read-only path.
constexpr size_t kMaxBatchChunk = 64;  // proofs per prover call of a batch, at most
struct WitnessPtrs {
    const fe* v[kMaxBatchChunk];
};
__global__ void k_gather_wires(const uint32_t* __restrict__ wire_vars, WitnessPtrs wit, size_t n, size_t num_inputs,
                               fe* __restrict__ wires_ev, fe* __restrict__ pi_poly, size_t pstride) {
    const size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= NW * n) return;
    const size_t p = blockIdx.y;
    const fe x = fe_load_ro(wit.v[p] + __ldg(wire_vars + t));
    fe_store(wires_ev + p * NW * n + t, x);
    if (t >= (NW - 1) * n && t - (NW - 1) * n < num_inputs) fe_store(pi_poly + p * pstride + (t - (NW - 1) * n), x);
}

// out[i] = n * (x_i - 1)   (inverted afterwards: L_1(x) / Z_H(x) = 1 / (n (x - 1)))
__global__ void k_l1_denominators(const fe* __restrict__ pts, size_t m, fe n_mont, fe* __restrict__ out) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= m) return;
    fe_store(out + i, FMUL(FSUB(fe_load_ro(pts + i), fe_one<Fr>()), n_mont));
}

// Batch inversion with ONE field inversion per block of 4096 elements (Montgomery's trick on two levels): every thread
// multiplies up its chunk of 16, the 256 chunk totals are scanned in shared memory (prefix and suffix products at once),
// thread 0 inverts the block total with the binary extended Euclid — a single lane, so its data-dependent branches have
// nobody to diverge from, far shorter than the 380 dependent products of a Fermat ladder (what a per-thread inversion
// costs whatever the batch size) — and the chunk inverses fan back out.  ~5 products per element.  Measured faster than
// a Fermat ladder per 16 elements, a one-lane Fermat per block, and block totals inverted on the host.
// data[i] <- 1 / data[i], or num[i] / data[i] (RATIO); zeros stay zero and do not disturb their neighbours.
constexpr int kInvThreads = 256, kInvChunk = 16, kInvBlock = kInvThreads * kInvChunk;
template <bool RATIO>
__global__ void __launch_bounds__(kInvThreads) k_block_inverse(const fe* __restrict__ num, fe* __restrict__ data,
                                                               fe* __restrict__ scratch, size_t n) {
    __shared__ fe pre[kInvThreads], suf[kInvThreads];
    __shared__ fe binv;
    const unsigned t = threadIdx.x;
    const size_t beg = ((size_t)blockIdx.x * kInvThreads + t) * kInvChunk;
    const size_t end = beg + kInvChunk < n ? beg + kInvChunk : n;
    const fe one = fe_one<Fr>();
    fe run = one;
    for (size_t i = beg; i < end; ++i) {
        fe_store(scratch + i, run);
        const fe d = fe_load(data + i);
        if (!fe_is_zero(d)) run = FMUL(run, d);
    }
    fe p = run, s = run;
    pre[t] = p;
    suf[t] = s;
    __syncthreads();
#pragma unroll 1
    for (unsigned off = 1; off < kInvThreads; off <<= 1) {
        fe pp = one, ss = one;
        if (t >= off) pp = pre[t - off];
        if (t + off < kInvThreads) ss = suf[t + off];
        __syncthreads();
        if (t >= off) p = FMUL(p, pp);
        if (t + off < kInvThreads) s = FMUL(s, ss);
        pre[t] = p;
        suf[t] = s;
        __syncthreads();
    }
    if (t == 0) binv = fe_inv_euclid<Fr>(pre[kInvThreads - 1]);
    __syncthreads();
    fe inv = binv;
    if (t > 0) inv = FMUL(inv, pre[t - 1]);
    if (t + 1 < kInvThreads) inv = FMUL(inv, suf[t + 1]);
    for (size_t i = end; i-- > beg;) {
        const fe d = fe_load(data + i);
        const bool zero = fe_is_zero(d);
        fe r = FMUL(inv, fe_load(scratch + i));
        if (RATIO) r = FMUL(fe_load_ro(num + i), r);
        fe_store(data + i, zero ? fe_zero() : r);
        if (!zero) inv = FMUL(inv, d);
    }
}

// ---- round 1 / 2 helpers -------------------------------------------------------------------------
// Per-proof scalars (blinders, challenges and what the host derives from them) reach the prover's kernels through
// `dyn`: a pointer into the context's device copy of ProofParams, so that the kernel ARGUMENTS are the same for every
// proof of a key and a round can be replayed as a CUDA graph.  dyn == nullptr: the by-value fields are used (link
// proofs, the stand-alone polynomial entry points).
// A batch of k proofs of one key runs every launch once over all k: the proof index is a grid index (blockIdx.y, or
// the first free one), each proof's data sits `*stride` elements after the previous proof's, and its scalars are the
// next ProofParams of the array (`dstride` = sizeof(ProofParams) in elements).  A single proof is the k = 1 case.
struct BlindArgs {
    fe b[3];
    int count;
    const fe* dyn;
};
// poly += (b0 + b1 X + ...) * (X^n - 1); block p: proof p
__global__ void k_blind(fe* poly, size_t n, BlindArgs a, size_t pstride, size_t dstride) {
    const int i = threadIdx.x;
    if (i >= a.count) return;
    poly += blockIdx.x * pstride;
    const fe b = a.dyn ? fe_load_ro(a.dyn + blockIdx.x * dstride + i) : a.b[i];
    fe_store(poly + i, FSUB(fe_load(poly + i), b));
    fe_store(poly + n + i, FADD(fe_load(poly + n + i), b));
}

// the five wire polynomials in one launch: thread (i, t) adds blinder t of wire i; block p: proof p
__global__ void k_blind_wires(fe* wpoly, size_t stride, size_t n, const fe* __restrict__ dyn /* [NW][2] */, size_t dstride) {
    const int i = threadIdx.x >> 1, t = threadIdx.x & 1;
    if (i >= NW) return;
    fe* poly = wpoly + ((size_t)blockIdx.x * NW + i) * stride;
    const fe b = fe_load_ro(dyn + blockIdx.x * dstride + 2 * i + t);
    fe_store(poly + t, FSUB(fe_load(poly + t), b));
    fe_store(poly + n + t, FADD(fe_load(poly + n + t), b));
}

// per row j: num = prod_i (w_ij + beta k_i w^j + gamma), den = prod_i (w_ij + beta sigma_ij + gamma); blockIdx.y: proof
__global__ void k_perm_num_den(const fe* __restrict__ wires, const fe* __restrict__ sig_evals,
                               const fe* __restrict__ dom, KArr k, const fe* __restrict__ beta_gamma, size_t dstride, size_t n,
                               fe* __restrict__ num, fe* __restrict__ den) {
    const size_t j = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n) return;
    wires += (size_t)blockIdx.y * NW * n;
    beta_gamma += blockIdx.y * dstride;
    num += (size_t)blockIdx.y * n;
    den += (size_t)blockIdx.y * n;
    const fe beta = fe_load_ro(beta_gamma), gamma = fe_load_ro(beta_gamma + 1);
    const fe bw = FMUL(beta, fe_load_ro(dom + j));
    fe a = fe_one<Fr>(), b = fe_one<Fr>();
#pragma unroll
    for (int i = 0; i < NW; ++i) {
        const fe t = FADD(fe_load_ro(wires + i * n + j), gamma);
        a = FMUL(a, FADD(t, FMUL(k.v[i], bw)));
        b = FMUL(b, FADD(t, FMUL(beta, fe_load_ro(sig_evals + i * n + j))));
    }
    fe_store(num + j, a);
    fe_store(den + j, b);
}

// segmented exclusive multiplicative scan, chunked: data[j] <- product of the elements before j in its segment of `seg`.
// A chunk never straddles two segments: thread t runs chunk t % cps of segment t / cps (cps = chunks per segment), so
// the chunk totals are again `cps`-long segments, one per proof.
__global__ void k_scan_mul_local(fe* __restrict__ data, size_t seg, size_t cps, size_t n_chunks, fe* __restrict__ totals) {
    const size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n_chunks) return;
    const size_t s = t / cps;
    const size_t beg = s * seg + (t - s * cps) * CH, seg_end = (s + 1) * seg;
    const size_t end = beg + CH < seg_end ? beg + CH : seg_end;
    fe run = fe_one<Fr>();
    for (size_t i = beg; i < end; ++i) {
        const fe v = fe_load(data + i);
        fe_store(data + i, run);
        run = FMUL(run, v);
    }
    fe_store(totals + t, run);
}
__global__ void k_scan_mul_apply(fe* __restrict__ data, size_t seg, size_t total, size_t cps, const fe* __restrict__ offs) {
    const size_t j = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= total) return;
    const size_t s = j / seg, jl = j - s * seg;
    if (jl < CH) return;  // the first chunk's offset is 1
    fe_store(data + j, FMUL(fe_load(data + j), fe_load_ro(offs + s * cps + jl / CH)));
}

// ---- Horner suffix scan: S[j] = sum_{i >= j} p[i] z^(i-j) -------------------------------------------
// S[0] = p(z) (evaluation) and S[1..] are the coefficients of p(X) / (X - z) (synthetic division).
// Batches (blockIdx.y = proof): the strides of HornerStrides below; H holds [proof][chunk].
__global__ void k_horner_local(const fe* __restrict__ p, size_t pstride, size_t len, fe z_val, const fe* __restrict__ z_dyn,
                               size_t dstride, fe* __restrict__ S, size_t sstride, fe* __restrict__ H) {
    const size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const size_t beg = t * CH;
    if (beg >= len) return;
    const size_t end = beg + CH < len ? beg + CH : len;
    const size_t q = blockIdx.y;
    p += q * pstride;
    if (S) S += q * sstride;
    const fe z = z_dyn ? fe_load_ro(z_dyn + q * dstride) : z_val;
    fe run = fe_zero();
    for (size_t i = end; i-- > beg;) {
        run = FADD(FMUL(run, z), fe_load_ro(p + i));
        if (S) fe_store(S + i, run);
    }
    fe_store(H + q * ((len + CH - 1) / CH) + t, run);
}
// batched evaluation-only variant: blockIdx.y selects the polynomial, blockIdx.z the proof
constexpr int kMaxEval = 10;
struct EvalArgs {
    const fe* p[kMaxEval];
    size_t pstride[kMaxEval];  // proof y's polynomial q: p[q] + y * pstride[q]
    fe* H[kMaxEval];
    size_t hstride;            // proof y's outputs: H[q] + y * hstride
    fe z[kMaxEval];
    uint32_t len[kMaxEval];
    const fe* dyn;   // z[] of this level in device memory, or null
    size_t dstride;  // proof y's z[]: dyn + y * dstride
};
__global__ void k_horner_local_batch(EvalArgs a) {
    const int q = blockIdx.y;
    const size_t y = blockIdx.z;
    const size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const size_t beg = t * CH, len = a.len[q];
    if (beg >= len) return;
    const size_t end = beg + CH < len ? beg + CH : len;
    const fe z = a.dyn ? fe_load_ro(a.dyn + y * a.dstride + q) : a.z[q];
    const fe* p = a.p[q] + y * a.pstride[q];
    fe run = fe_zero();
    for (size_t i = end; i-- > beg;) run = FADD(FMUL(run, z), fe_load_ro(p + i));
    fe_store(a.H[q] + y * a.hstride + t, run);
}
// S[j] += z^(chunk_end - j) * T[chunk + 1], one thread per element; zpow[e] = z^e for e = 1..CH; blockIdx.y: proof
struct ZPow {
    fe v[CH + 1];
};
__global__ void k_horner_apply(fe* __restrict__ S, size_t sstride, size_t len, ZPow zp, const fe* __restrict__ zp_dyn,
                               size_t dstride, const fe* __restrict__ T, size_t n_chunks) {
    const size_t j = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const size_t t = j / CH;
    if (j >= len || t + 1 >= n_chunks) return;  // the last chunk has no carry
    const size_t q = blockIdx.y;
    S += q * sstride;
    T += q * n_chunks;
    const size_t e = (t + 1) * CH - j;
    const fe ze = zp_dyn ? fe_load_ro(zp_dyn + q * dstride + e) : zp.v[e];
    fe_store(S + j, FADD(fe_load(S + j), FMUL(ze, fe_load_ro(T + t + 1))));
}

// ---- round 3: quotient over nc cosets s_j * H_n of the 8n-th roots' coset g * H_8n ---------------------
// The reference evaluates the quotient on all of g * H_8n (8n points, the next power of two above its
// degree 5n + 7) and interpolates with one size-8n inverse FFT.  g * H_8n is the union of the 8 cosets
// s_j * H_n, s_j = g * w_8n^j, and t(X) = sum_k X^(kn) t_k(X) (deg t_k < n) restricted to coset j is
// u_j = sum_k c_j^k t_k with c_j = s_j^n: nc = 6 cosets (6n > 5n + 7 points) determine t.  So every
// polynomial is evaluated on 6 cosets with size-n transforms (after folding X^n -> c_j), the quotient
// kernel runs on 6n points, and t comes back from 6 size-n inverse transforms and one 6 x 6
// inverse-Vandermonde combination per coefficient index — the same coefficients, 25 % fewer points and
// 16 instead of 19 butterfly levels.  Layout of every table: [coset j][h], point s_j * w_n^h.
struct CosetConsts {
    fe cn[8];  // c_j = s_j^n
};
// dst[(p * nc + j) * n + i] = (a_p[i] + c_j * a_p[n + i]) * s_j^i : input of the size-n transform that
// evaluates polynomial p (len <= 2n coefficients, `src_stride` apart) on coset j
__global__ void k_coset_fold(const fe* __restrict__ src, size_t src_stride, size_t len, size_t n, int nc,
                             CosetConsts cc, const fe* __restrict__ cscale, fe* __restrict__ dst) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int j = blockIdx.y;
    const fe* a = src + (size_t)blockIdx.z * src_stride;
    fe v = fe_load_ro(a + i);
    if (n + i < len) v = FADD(v, FMUL(cc.cn[j], fe_load_ro(a + n + i)));
    v = FMUL(v, fe_load_ro(cscale + (size_t)j * n + i));
    fe_store(dst + ((size_t)blockIdx.z * nc + j) * n + i, v);
}

constexpr int kMaxCosets = 8;
struct CombineArgs {
    fe minv[kMaxCosets * kMaxCosets];  // inverse of the Vandermonde matrix V[j][k] = c_j^k, row-major [k][j]
};
// in place: q[j * n + i] holds (n^-1-scaled) coefficient i of u_j(s_j X); afterwards q[k * n + i] = t_k[i];
// blockIdx.y: proof (NC * n elements each)
template <int NC>
__global__ void k_coset_combine(fe* __restrict__ q, size_t n, const fe* __restrict__ cscale_inv, CombineArgs a) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    q += (size_t)blockIdx.y * NC * n;
    fe u[NC];
#pragma unroll
    for (int j = 0; j < NC; ++j) u[j] = FMUL(fe_load(q + (size_t)j * n + i), fe_load_ro(cscale_inv + (size_t)j * n + i));
#pragma unroll 1
    for (int k = 0; k < NC; ++k) {
        fe acc = FMUL(a.minv[k * NC], u[0]);
#pragma unroll
        for (int j = 1; j < NC; ++j) acc = FADD(acc, FMUL(a.minv[k * NC + j], u[j]));
        fe_store(q + (size_t)k * n + i, acc);
    }
}

struct QuotArgs {
    const fe* sel;   // 13 x m resident coset evaluations
    const fe* sig;   // 5 x m
    const fe* ext;   // per proof NW x m: wires 0..4
    const fe* pi;    // per proof m: public-input polynomial
    const fe* zext;  // per proof m: z
    const fe* pts;   // m evaluation points s_j * w_n^h
    const fe* l1_inv;  // 1 / (n (x_i - 1))
    fe* out;         // per proof m
    size_t m;        // nc * n
    unsigned log_n;
    KArr k;
    const fe* chal;  // device: beta, gamma, alpha, alpha^2
    size_t dstride;  // next proof's chal[]
    fe zh_inv[8];    // 1 / (c_j - 1)
};
// k_quotient chains ~60 field products; fully unrolled it is ~180 KB of code and starves on the
// instruction cache ("no instruction" stalls; an out-of-line multiplier was slower still, through
// stack traffic).  The per-wire loops are therefore kept rolled.  blockIdx.y: proof.
__global__ void __launch_bounds__(128) k_quotient(QuotArgs a) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= a.m) return;
    const size_t m = a.m, pr = blockIdx.y;
    const fe* ext = a.ext + pr * NW * m;
    const fe* zext = a.zext + pr * m;
    const fe* chal = a.chal + pr * a.dstride;
    const fe beta = fe_load_ro(chal), gamma = fe_load_ro(chal + 1);
    fe w[NW];
#pragma unroll
    for (int j = 0; j < NW; ++j) w[j] = fe_load_ro(ext + j * m + i);
    // gate: q_c + pi + sum q_lc w + q_mul0 w0 w1 + q_mul1 w2 w3 + q_ecc w0..w4 + sum q_hash w^5 - q_o w4
    fe acc = FADD(fe_load_ro(a.sel + 11 * m + i), fe_load_ro(a.pi + pr * m + i));
#pragma unroll 1
    for (int j = 0; j < 4; ++j) {
        acc = FADD(acc, FMUL(fe_load_ro(a.sel + j * m + i), w[j]));
        const fe w2 = fe_sqr<Fr>(w[j]);
        acc = FADD(acc, FMUL(fe_load_ro(a.sel + (6 + j) * m + i), FMUL(fe_sqr<Fr>(w2), w[j])));
    }
    const fe w01 = FMUL(w[0], w[1]), w23 = FMUL(w[2], w[3]);
    acc = FADD(acc, FMUL(fe_load_ro(a.sel + 4 * m + i), w01));
    acc = FADD(acc, FMUL(fe_load_ro(a.sel + 5 * m + i), w23));
    acc = FADD(acc, FMUL(fe_load_ro(a.sel + 12 * m + i), FMUL(FMUL(w01, w23), w[4])));
    acc = FSUB(acc, FMUL(fe_load_ro(a.sel + 10 * m + i), w[4]));
    // permutation: alpha * ( z prod(w + beta k x + gamma) - z(wx) prod(w + beta sigma + gamma) )
    const fe zx = fe_load_ro(zext + i);
    const size_t nmask = ((size_t)1 << a.log_n) - 1;
    const fe zxw = fe_load_ro(zext + ((i & ~nmask) | ((i + 1) & nmask)));  // z(w x): next point of the same coset
    const fe bx = FMUL(beta, fe_load_ro(a.pts + i));
    fe p1 = zx, p2 = zxw;
#pragma unroll 1
    for (int j = 0; j < NW; ++j) {
        const fe t = FADD(w[j], gamma);
        p1 = FMUL(p1, FADD(t, FMUL(a.k.v[j], bx)));
        p2 = FMUL(p2, FADD(t, FMUL(beta, fe_load_ro(a.sig + j * m + i))));
    }
    acc = FADD(acc, FMUL(fe_load_ro(chal + 2), FSUB(p1, p2)));
    acc = FMUL(acc, a.zh_inv[i >> a.log_n]);
    // alpha^2 (z - 1) L1(x) / Z_H(x)
    acc = FADD(acc, FMUL(FMUL(fe_load_ro(chal + 3), FSUB(zx, fe_one<Fr>())), fe_load_ro(a.l1_inv + i)));
    fe_store(a.out + pr * m + i, acc);
}

// flag bit 0: a coefficient above `deg` is non-zero; bit 1: coefficient `deg` is zero; blockIdx.y: proof (its m
// coefficients and its own flag)
__global__ void k_check_degree(const fe* __restrict__ q, size_t deg, size_t m, uint32_t* flag) {
    const size_t i = deg + (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= m) return;
    q += (size_t)blockIdx.y * m;
    flag += blockIdx.y;
    const bool zero = fe_is_zero(fe_load_ro(q + i));
    if (i == deg) {
        if (zero) atomicOr(flag, 2u);
    } else if (!zero) {
        atomicOr(flag, 1u);
    }
}

// ---- link proofs: one descriptor per item, blockIdx.y = item ----------------------------------------------------
struct LinkDesc {
    fe g, root0;        // generator of the layout's 2^alignment roots of unity, and the group's first root g^offset
    uint64_t roots_at;  // where the item's roots start in the batch's root array
    uint64_t size;      // roots in the group
    uint64_t q_len;     // quotient coefficients: len - size
    uint64_t pad;
};

// roots[roots_at + i] = root0 * g^i, i < size
__global__ void k_link_roots(const LinkDesc* __restrict__ d, fe* __restrict__ roots) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const LinkDesc* it = d + blockIdx.y;
    if (i >= it->size) return;
    fe base = it->g, acc = it->root0;
    for (size_t e = i; e; e >>= 1) {
        if (e & 1) acc = FMUL(acc, base);
        base = fe_sqr<Fr>(base);
    }
    fe_store(roots + it->roots_at + i, acc);
}

// out[y * N + j] = prod_i (x_j - roots_y[i]), x_j = g * w^j the j-th point of the coset g * H_N (tw[k] = w^k, k < N/2),
// for the items y of one transform size N, each with its roots from its descriptor
__global__ void k_vanishing_on_coset_batch(const fe* __restrict__ tw, size_t N, fe g, const fe* __restrict__ roots,
                                           const LinkDesc* __restrict__ d, fe* __restrict__ out) {
    const size_t j = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= N) return;
    const LinkDesc* it = d + blockIdx.y;
    const size_t half = N >> 1;
    fe wj = fe_load_ro(tw + (j < half ? j : j - half));
    if (j >= half) wj = fe_neg<Fr>(wj);
    const fe x = FMUL(g, wj);
    const fe* r = roots + it->roots_at;
    const size_t count = it->size;
    fe acc = fe_one<Fr>();
    for (size_t i = 0; i < count; ++i) acc = FMUL(acc, FSUB(x, fe_load_ro(r + i)));
    fe_store(out + blockIdx.y * N + j, acc);
}

// flag[y] |= 1 when item y's coefficients [q_len_y, m) are not all zero (q + y * m): the division was not exact
__global__ void k_check_zero_tail(const fe* __restrict__ q, size_t m, const LinkDesc* __restrict__ d, uint32_t* flag) {
    const size_t i = d[blockIdx.y].q_len + (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= m) return;
    if (!fe_is_zero(fe_load_ro(q + blockIdx.y * m + i))) atomicOr(flag + blockIdx.y, 1u);
}


// ---- element-wise Fr vector primitives (the collaborative prover's share arithmetic) ------------------------------
// out[i] = a[i] (op) b[i]  or  a[i] (op) b[0] when b is a scalar; op: 0 add, 1 sub, 2 mul
__global__ void k_fr_vec_op(int op, const fe* __restrict__ a, const fe* __restrict__ b, int b_scalar, size_t n, fe* __restrict__ out) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const fe x = fe_load(a + i), y = fe_load(b + (b_scalar ? 0 : i));
    fe r;
    switch (op) {
        case 0: r = FADD(x, y); break;
        case 1: r = FSUB(x, y); break;
        default: r = FMUL(x, y); break;
    }
    fe_store(out + i, r);
}


// t_i = quot[i(n+2) .. ) - b_{i-1} + b_i X^(n+2)   (the last chunk has n coefficients); blockIdx.z: proof
__global__ void k_split_quotient(const fe* __restrict__ quot, size_t qstride, size_t n, size_t stride,
                                 const fe* __restrict__ dyn /* b[4] */, size_t dstride, fe* __restrict__ out) {
    const size_t j = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int i = blockIdx.y;
    if (j >= n + 3) return;
    quot += blockIdx.z * qstride;
    dyn += blockIdx.z * dstride;
    out += (size_t)blockIdx.z * NW * stride;
    const size_t len = i < NW - 1 ? n + 2 : n;
    fe v = j < len ? fe_load_ro(quot + (size_t)i * (n + 2) + j) : fe_zero();
    if (j == 0 && i > 0) v = FSUB(v, fe_load_ro(dyn + i - 1));
    if (j == n + 2 && i < NW - 1) v = fe_load_ro(dyn + i);
    fe_store(out + (size_t)i * stride + j, v);
}

// ---- round 5: linear combination of polynomials -------------------------------------------------------
constexpr int kMaxLin = 32;
struct LinArgs {
    const fe* p[kMaxLin];
    uint32_t pstride[kMaxLin];  // proof y's term t: p[t] + y * pstride[t] (0: a polynomial of the key)
    uint32_t len[kMaxLin];
    fe s[kMaxLin];
    int count;
    const fe* dyn;  // s[] in device memory, or null
    size_t dstride; // proof y's s[]: dyn + y * dstride
};
// blockIdx.y: proof (output `ostride` apart)
__global__ void k_lincomb(LinArgs a, size_t out_len, fe* __restrict__ out, size_t ostride) {
    const size_t j = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= out_len) return;
    const size_t y = blockIdx.y;
    fe acc = fe_zero();
    for (int t = 0; t < a.count; ++t)
        if (j < a.len[t])
            acc = FADD(acc, FMUL(a.dyn ? fe_load_ro(a.dyn + y * a.dstride + t) : a.s[t], fe_load_ro(a.p[t] + y * a.pstride[t] + j)));
    fe_store(out + y * ostride + j, acc);
}

// ---- per-proof scalars ------------------------------------------------------------------------------------
// Everything a proof's kernels need that is not a function of (context, proving key): blinders, Fiat–Shamir challenges
// and the host-side values derived from them.  The host fills the pinned copy between rounds; each round's first
// operation copies it to the device copy the kernels read (see `dyn` above).
constexpr int kLevels = 8;  // levels of the chunked Horner scans: CH^8 = 2^32 coefficients
struct OpenParams {
    fe z[kLevels];     // the point raised to CH^level
    ZPow zp[kLevels];  // powers 0..CH of z[level]
};
struct ProofParams {
    fe blind_w[NW][2];             // round 1
    fe chal[4];                    // beta, gamma (round 2), alpha, alpha^2 (round 3)
    fe blind_z[4];                 // 3 used
    fe blind_q[4];                 // round 3
    fe eval_z[kLevels][kMaxEval];  // round 4
    fe lin_s[kMaxLin];             // round 5
    OpenParams open[2];            // zeta, zeta * w
};

struct LinkParams {  // the same for a link proof
    fe lin_s[4];      // 1, -Z_D(eta)
    OpenParams open;  // eta
};

inline unsigned grid_for(size_t n, unsigned bs) { return (unsigned)((n + bs - 1) / bs); }

}  // namespace

// data[i] <- 1 / data[i] (num == nullptr) or num[i] / data[i]; enqueue only.  scratch: n elements.
void batch_inverse_enqueue(const fe* num, fe* data, fe* scratch, size_t n, cudaStream_t st) {
    if (num) B200_LAUNCH(k_block_inverse<true>, grid_for(n, kInvBlock), kInvThreads, 0, st)(num, data, scratch, n);
    else B200_LAUNCH(k_block_inverse<false>, grid_for(n, kInvBlock), kInvThreads, 0, st)(nullptr, data, scratch, n);
}

// ---------------------------------------------------------------------------------------------
// host-side structures
// ---------------------------------------------------------------------------------------------
struct ProvingKey {
    uint64_t id = g_object_ids.fetch_add(1);  // never reused: what a context's captured graphs are keyed by
    unsigned log_n = 0;
    size_t n = 0, m = 0, num_inputs = 0;
    KArr k;
    const Bases* srs = nullptr;
    fe *sel_coeffs = nullptr, *sig_coeffs = nullptr, *sig_evals = nullptr;
    fe *ce_sel = nullptr, *ce_sig = nullptr;
    fe *dom = nullptr, *coset_pts = nullptr, *l1_inv = nullptr;
    // quotient domain: nc cosets s_j * H_n, m = nc * n points (see "round 3" above)
    int nc = 0;
    fe *cscale = nullptr, *cscale_inv = nullptr;  // s_j^i and s_j^-i, [j][i]
    CosetConsts cc;
    CombineArgs comb;
    fe zh_inv[8];
    fe group_gen;
    g1_affine sel_comms[NS], sig_comms[NW];
    // keys made from the wiring (b200_plonk_preprocess_wiring) keep it: the variable on every wire position (device, NW x n),
    // the length of the witness vector, and the variables of the public inputs (host: the transcript starts with them)
    uint32_t* wire_vars = nullptr;
    size_t num_vars = 0;
    std::vector<uint32_t> pub_vars;
    ~ProvingKey() {
        for (fe* p : {sel_coeffs, sig_coeffs, sig_evals, ce_sel, ce_sig, dom, coset_pts, l1_inv, cscale, cscale_inv})
            if (p) cudaFree(p);
        if (wire_vars) cudaFree(wire_vars);
    }
};

// inverse of the nc x nc matrix a (row-major) over Fr by Gauss–Jordan elimination (host, set-up time)
static bool host_mat_inverse(const fe* a, int nc, fe* out) {
    const fe one = fe_one<Fr>(), zero = fe_zero();
    std::vector<fe> m((size_t)nc * 2 * nc);
    for (int r = 0; r < nc; ++r)
        for (int c = 0; c < nc; ++c) {
            m[(size_t)r * 2 * nc + c] = a[r * nc + c];
            m[(size_t)r * 2 * nc + nc + c] = r == c ? one : zero;
        }
    for (int col = 0; col < nc; ++col) {
        int piv = -1;
        for (int r = col; r < nc && piv < 0; ++r)
            if (!fe_is_zero(m[(size_t)r * 2 * nc + col])) piv = r;
        if (piv < 0) return false;
        for (int c = 0; c < 2 * nc; ++c) std::swap(m[(size_t)col * 2 * nc + c], m[(size_t)piv * 2 * nc + c]);
        const fe iv = fe_inv<Fr>(m[(size_t)col * 2 * nc + col]);
        for (int c = 0; c < 2 * nc; ++c) m[(size_t)col * 2 * nc + c] = FMUL(m[(size_t)col * 2 * nc + c], iv);
        for (int r = 0; r < nc; ++r) {
            if (r == col) continue;
            const fe f = m[(size_t)r * 2 * nc + col];
            if (fe_is_zero(f)) continue;
            for (int c = 0; c < 2 * nc; ++c)
                m[(size_t)r * 2 * nc + c] = FSUB(m[(size_t)r * 2 * nc + c], FMUL(f, m[(size_t)col * 2 * nc + c]));
        }
    }
    for (int r = 0; r < nc; ++r)
        for (int c = 0; c < nc; ++c) out[r * nc + c] = m[(size_t)r * 2 * nc + nc + c];
    return true;
}

static fe host_pow(fe a, uint64_t e) {
    fe r = fe_one<Fr>();
    while (e) {
        if (e & 1) r = FMUL(r, a);
        a = fe_sqr<Fr>(a);
        e >>= 1;
    }
    return r;
}
static fe host_from_u64(uint64_t v) {
    fe x = fe_zero();
    x.l[0] = (uint32_t)v;
    x.l[1] = (uint32_t)(v >> 32);
    return fe_to_mont<Fr>(x);
}

// Runs the enclosed launches on the context's low-priority stream (b200_init), ordered after what is
// already queued on `st` and before what `st` gets next: for the long throughput-bound kernels, so that
// other contexts' short kernels are scheduled ahead of them.
struct HeavyScope {
    Context* c;
    cudaStream_t st, run;
    HeavyScope(Context* c_, cudaStream_t st_) : c(c_), st(st_), run(c_->heavy_plonk ? c_->heavy : st_) {
        if (c->heavy_plonk) {
            cudaEventRecord(c->hv_fork, st);
            cudaStreamWaitEvent(run, c->hv_fork, 0);
        }
    }
    ~HeavyScope() {
        if (c->heavy_plonk) {
            cudaEventRecord(c->hv_join, run);
            cudaStreamWaitEvent(st, c->hv_join, 0);
        }
    }
};

// exclusive product scan of k segments of `seg` elements (data[0..k*seg)) in place, each segment on its own;
// scratch >= k * (seg/CH + seg/CH^2 + 2*CH + 8) elements
static void scan_mul_exclusive(fe* data, size_t seg, unsigned k, fe* scratch, cudaStream_t st) {
    const size_t cps = (seg + CH - 1) / CH, n1 = cps * k;
    B200_LAUNCH(k_scan_mul_local, grid_for(n1, 128), 128, 0, st)(data, seg, cps, n1, scratch);
    if (cps > 1) {
        scan_mul_exclusive(scratch, cps, k, scratch + n1, st);
        B200_LAUNCH(k_scan_mul_apply, grid_for(seg * k, 256), 256, 0, st)(data, seg, seg * k, cps, scratch);
    }
}

// k Horner scans at once: proof q's polynomial is p + q * p, its suffix sums S + q * s, its p(z) out_total + q * out,
// its point and powers dyn + q * dyn (elements)
struct HornerStrides {
    unsigned k = 1;
    size_t p = 0, s = 0, out = 0, dyn = 0;
};

// Horner suffix scan; S may be null (evaluation only).  The value p(z) ends up at out_total (device).
// scratch >= k * 2 * (len/CH + len/CH^2 + 2*CH + 8) elements
// `dyn` (device, or null): the point and its powers per level come from there instead of `z` (see ProofParams).
static void horner_suffix(const fe* p, size_t len, fe z, fe* S, fe* out_total, fe* scratch, cudaStream_t st,
                          const OpenParams* dyn = nullptr, HornerStrides b = {}, int level = 0) {
    const size_t n1 = (len + CH - 1) / CH;
    fe* H = scratch;           // [proof][n1]
    fe* T = scratch + b.k * n1;
    B200_LAUNCH(k_horner_local, dim3(grid_for(n1, 128), b.k), 128, 0, st)(p, b.p, len, z, dyn ? &dyn->z[level] : nullptr, b.dyn,
                                                                          S, b.s, H);
    if (n1 == 1) {
        if (b.k == 1) cudaMemcpyAsync(out_total, H, sizeof(fe), cudaMemcpyDeviceToDevice, st);
        else cudaMemcpy2DAsync(out_total, b.out * sizeof(fe), H, sizeof(fe), sizeof(fe), b.k, cudaMemcpyDeviceToDevice, st);
        return;
    }
    const fe zc = dyn ? z : host_pow(z, CH);
    HornerStrides next = b;
    next.p = next.s = n1;
    horner_suffix(H, n1, zc, S ? T : nullptr, out_total, scratch + 2 * b.k * n1, st, dyn, next, level + 1);
    if (S) {
        ZPow zp{};
        if (!dyn) {
            zp.v[0] = fe_one<Fr>();
            for (int e = 1; e <= CH; ++e) zp.v[e] = FMUL(zp.v[e - 1], z);
        }
        B200_LAUNCH(k_horner_apply, dim3(grid_for(len, 256), b.k), 256, 0, st)(S, b.s, len, zp, dyn ? dyn->zp[level].v : nullptr,
                                                                               b.dyn, T, n1);
    }
}

// p_q(z_q) for up to kMaxEval polynomials, written to out[q], for k proofs at once: proof y's polynomial q is
// polys[q] + y * pstrides[q] (pstrides may be null: one proof), its results go to out + y * ostride;
// scratch: k * count * (max_len/CH + max_len/CH^2 + 2*CH + 16)
// `dyn_z` (device, or null): [level][kMaxEval] evaluation points, points[q]^(CH^level), proof y's `dstride` elements
// after proof 0's; `points` is unused then.
static void eval_batch(const fe* const* polys, const size_t* lens, const fe* points, int count, fe* out, fe* scratch,
                       cudaStream_t st, const fe (*dyn_z)[kMaxEval] = nullptr, unsigned k = 1, const size_t* pstrides = nullptr,
                       size_t ostride = 0, size_t dstride = 0) {
    EvalArgs a;
    size_t cur_len[kMaxEval], max_len = 0;
    for (int q = 0; q < count; ++q) {
        a.p[q] = polys[q];
        a.pstride[q] = pstrides ? pstrides[q] : 0;
        a.z[q] = dyn_z ? fe_zero() : points[q];
        cur_len[q] = lens[q];
        max_len = lens[q] > max_len ? lens[q] : max_len;
    }
    a.dstride = dstride;
    // two disjoint regions per polynomial (levels alternate A, B, A, ...): a level reads one and
    // writes the other
    const size_t region_a = max_len / CH + 2, region_b = max_len / CH / CH + CH + 2;
    const size_t per_poly = region_a + region_b;
    int level = 0;
    while (true) {
        bool last = true;
        size_t max_chunks = 0;
        for (int q = 0; q < count; ++q) {
            const size_t n1 = (cur_len[q] + CH - 1) / CH;
            if (n1 > 1) last = false;
            max_chunks = n1 > max_chunks ? n1 : max_chunks;
        }
        for (int q = 0; q < count; ++q) {
            a.len[q] = (uint32_t)cur_len[q];
            // levels alternate between the two halves of each polynomial's scratch slice
            a.H[q] = last ? out + q : scratch + (size_t)q * per_poly + (level & 1 ? region_a : 0);
        }
        a.hstride = last ? ostride : (size_t)count * per_poly;
        a.dyn = dyn_z ? &dyn_z[level][0] : nullptr;
        B200_LAUNCH(k_horner_local_batch, dim3(grid_for(max_chunks, 64), count, k), 64, 0, st)(a);
        if (last) break;
        for (int q = 0; q < count; ++q) {
            a.p[q] = a.H[q];
            a.pstride[q] = a.hstride;
            if (!dyn_z) a.z[q] = host_pow(a.z[q], CH);
            cur_len[q] = (cur_len[q] + CH - 1) / CH;
        }
        ++level;
    }
}

// The prover's device workspace for k proofs: every region holds the k proofs' copies one after the other (proof p's
// wire polynomials at wpoly + p * NW * S, its quotient at quot + p * m, ...), so that each step is one launch over
// all k with a uniform stride.  pi_poly sits directly behind the k * NW wire polynomials, and in `ext` the k public-input
// evaluations directly behind the wires': one batch of (NW + 1) k polynomials for the transforms, k * NW (no public
// input) for the commitments.  With k = 1 this is the single prover's layout.
struct Workspace {
    fe *wires_ev, *wpoly, *pi_poly, *zpoly, *num, *den, *tmp, *scan, *ext, *zext, *quot, *split, *lin, *sdiv, *hscr, *escr, *evals;
    uint32_t* flag;  // one per proof
    size_t S;  // stride of the (n + 3)-coefficient polynomials
};
constexpr size_t kEvalSlots = 32;  // per proof in `evals`: the 2 NW evaluations, then the two opening totals at 16, 17
static size_t workspace_elems(size_t n, unsigned k) {
    const size_t S = n + 4, m = 8 * n;
    return k * (NW * n + NW * S + S + S + 3 * n + (2 * (n / CH) + 4 * CH + 64) + 7 * m + m + NW * S + S + 2 * (S + 8) +
                4 * (S / CH + 4 * CH + 64) + kMaxEval * (S / CH + S / CH / CH + 2 * CH + 16) + kEvalSlots) +
           (k + 7) / 8 + 8;
}
static Workspace carve(fe* base, size_t n, unsigned k) {
    Workspace w;
    const size_t S = n + 4, m = 8 * n;
    w.S = S;
    fe* p = base;
    w.wires_ev = p; p += k * NW * n;
    w.wpoly = p; p += k * NW * S;
    w.pi_poly = p; p += k * S;
    w.zpoly = p; p += k * S;
    w.num = p; p += k * n;
    w.den = p; p += k * n;
    w.tmp = p; p += k * n;
    w.scan = p; p += k * (2 * (n / CH) + 4 * CH + 64);  // all levels of the product scan: n / CH * (1 + 1/CH + ...)
    w.ext = p; p += k * (NW + 1) * m;
    w.zext = p; p += k * m;
    w.quot = p; p += k * m;
    w.split = p; p += k * NW * S;
    w.lin = p; p += k * S;
    w.sdiv = p; p += k * 2 * (S + 8);
    w.hscr = p; p += k * 4 * (S / CH + 4 * CH + 64);
    w.escr = p; p += k * kMaxEval * (S / CH + S / CH / CH + 2 * CH + 16);
    w.evals = p; p += k * kEvalSlots;
    w.flag = reinterpret_cast<uint32_t*>(p);
    return w;
}

// `count` commitments to polynomials `stride` coefficients apart, in one batched MSM
static int commit_batch(Context* c, const ProvingKey* pk, const fe* d_coeffs, size_t len, size_t stride,
                        unsigned count, g1_affine* out) {
    std::vector<int> inf(count);
    int rc = msm_device_batch(pk->srs, 0, d_coeffs, len, stride, count, /*montgomery=*/1, &c->msm, c->stream, out, inf.data());
    if (rc != B200_OK) return rc;
    for (unsigned i = 0; i < count; ++i)
        if (inf[i]) std::memset(&out[i], 0, sizeof(out[i]));
    return B200_OK;
}

static int alloc_fe(fe** p, size_t count) {
    cudaError_t e = cudaMalloc(p, count * sizeof(fe));
    if (e != cudaSuccess) return cuda_fail(e, "cudaMalloc(proving key)");
    return B200_OK;
}

// Evaluations of `count` polynomials (`len` <= 2n coefficients each, `src_stride` apart) on the nc cosets
// of the quotient domain: dst[(p * nc + j) * n + h] = poly_p(s_j * w_n^h).  scratch: count * nc * n elements.
static int coset_evals(const ProvingKey* pk, const Domain* dn, const fe* src, size_t src_stride, size_t len,
                       unsigned count, fe* dst, fe* scratch, cudaStream_t st) {
    const size_t n = pk->n;
    if (len > 2 * n) {
        set_error("coset_evals: polynomial longer than 2n");
        return B200_ERR_INVALID;
    }
    B200_LAUNCH(k_coset_fold, dim3(grid_for(n, 256), (unsigned)pk->nc, count), 256, 0, st)(src, src_stride, len, n, pk->nc, pk->cc,
                                                                                 pk->cscale, dst);
    return ntt_device(dn, dst, scratch, /*inverse=*/0, /*coset=*/0, count * (unsigned)pk->nc, n, st);
}

// The copy permutation comes from the caller (h_perm) or, with h_perm null, is derived on the device from the wiring
// (h_wire_vars, num_vars), which the key then keeps.
static int preprocess(Context* c, const Bases* srs, unsigned log_n, size_t num_inputs, const fe* h_selectors,
                      const uint64_t* h_perm, const uint32_t* h_wire_vars, size_t num_vars, const fe* h_k, ProvingKey** out) {
    const size_t n = (size_t)1 << log_n;
    // 6 cosets (6n > 5n + 7 points) from n = 16 on; all 8 for the tiny domains, where 6n would not exceed
    // the quotient's degree by enough to keep the degree check meaningful.  Six cosets determine t for a satisfied
    // witness but do not decide satisfaction: the degree check misses violations of degree <= 7 on H, which prove()'s
    // self-check at zeta refuses (DESIGN §4)
    const int nc = log_n >= 4 ? 6 : 8;
    const size_t m = (size_t)nc * n;
    if (log_n < 2 || log_n + 3 > 28) {
        set_error("preprocess: log_n out of range");
        return B200_ERR_INVALID;
    }
    if (srs->n < n + 3) {
        set_error("preprocess: SRS shorter than n + 3 (MAX_SRS_DEGREE rule, srs.rs:44-47)");
        return B200_ERR_INVALID;
    }
    if (num_inputs > n) return B200_ERR_INVALID;
    cudaStream_t st = c->stream;
    ProvingKey* pk = new ProvingKey();
    pk->log_n = log_n;
    pk->n = n;
    pk->m = m;
    pk->nc = nc;
    pk->num_inputs = num_inputs;
    pk->srs = srs;
    for (int i = 0; i < NW; ++i) pk->k.v[i] = h_k[i];
    int rc;
    Domain* dn = nullptr;
    if ((rc = get_domain(c, log_n, &dn)) != B200_OK) {
        delete pk;
        return rc;
    }
    pk->group_gen = dn->group_gen;
    uint64_t* d_perm = nullptr;
    auto fail = [&](int code) {
        if (d_perm) cudaFree(d_perm);
        delete pk;
        return code;
    };
    if ((rc = alloc_fe(&pk->sel_coeffs, NS * n)) || (rc = alloc_fe(&pk->sig_coeffs, NW * n)) ||
        (rc = alloc_fe(&pk->sig_evals, NW * n)) || (rc = alloc_fe(&pk->ce_sel, NS * m)) ||
        (rc = alloc_fe(&pk->ce_sig, NW * m)) || (rc = alloc_fe(&pk->dom, n)) || (rc = alloc_fe(&pk->coset_pts, m)) ||
        (rc = alloc_fe(&pk->l1_inv, m)) || (rc = alloc_fe(&pk->cscale, m)) || (rc = alloc_fe(&pk->cscale_inv, m)))
        return fail(rc);
    if (cudaMalloc(&d_perm, NW * n * 8) != cudaSuccess) return fail(B200_ERR_CUDA);
    if ((rc = c->ntt_scratch.reserve((size_t)NS * m * sizeof(fe))) != B200_OK) return fail(rc);
    fe* scratch = reinterpret_cast<fe*>(c->ntt_scratch.p);

    const fe one = fe_one<Fr>();
    const fe g = fe_from_u32<Fr>(5);
    fill_powers(pk->dom, n, dn->group_gen, one, st);
    {
        const fe w8n = host_root_of_unity(log_n + 3);
        fe vand[kMaxCosets * kMaxCosets];
        for (int j = 0; j < nc; ++j) {
            const fe sj = FMUL(g, host_pow(w8n, (uint64_t)j));  // s_j = g * w_8n^j
            const fe cj = host_pow(sj, n);                       // x^n on the whole coset
            pk->cc.cn[j] = cj;
            pk->zh_inv[j] = fe_inv<Fr>(FSUB(cj, one));
            fe pw = one;
            for (int k = 0; k < nc; ++k) {
                vand[j * nc + k] = pw;
                pw = FMUL(pw, cj);
            }
            fill_powers(pk->coset_pts + (size_t)j * n, n, dn->group_gen, sj, st);  // s_j * w_n^h
            fill_powers(pk->cscale + (size_t)j * n, n, sj, one, st);               // s_j^i
            fill_powers(pk->cscale_inv + (size_t)j * n, n, fe_inv<Fr>(sj), one, st);
        }
        for (int j = nc; j < 8; ++j) {
            pk->cc.cn[j] = fe_zero();
            pk->zh_inv[j] = fe_zero();
        }
        if (!host_mat_inverse(vand, nc, pk->comb.minv)) {
            set_error("preprocess: singular coset Vandermonde matrix");
            return fail(B200_ERR_INVALID);
        }
    }
    B200_LAUNCH(k_l1_denominators, grid_for(m, 256), 256, 0, st)(pk->coset_pts, m, host_from_u64(n), pk->l1_inv);
    batch_inverse_enqueue(nullptr, pk->l1_inv, pk->ce_sel /*scratch, overwritten below*/, m, st);

    // selectors: evaluations -> coefficients -> commitments
    cudaMemcpyAsync(pk->sel_coeffs, h_selectors, NS * n * sizeof(fe), cudaMemcpyHostToDevice, st);
    if ((rc = ntt_device(dn, pk->sel_coeffs, scratch, 1, 0, NS, n, st)) != B200_OK) return fail(rc);
    // sigmas: permutation -> evaluations (kept for the grand product) -> coefficients
    if (h_perm) {
        cudaMemcpyAsync(d_perm, h_perm, NW * n * 8, cudaMemcpyHostToDevice, st);
    } else {
        if (cudaMalloc(&pk->wire_vars, NW * n * sizeof(uint32_t)) != cudaSuccess) return fail(cuda_fail(cudaGetLastError(), "cudaMalloc(wiring)"));
        cudaMemcpyAsync(pk->wire_vars, h_wire_vars, NW * n * sizeof(uint32_t), cudaMemcpyHostToDevice, st);
        if ((rc = wiring_permutation(pk->wire_vars, NW * n, num_vars, d_perm, st)) != B200_OK) return fail(rc);
        pk->num_vars = num_vars;
        pk->pub_vars.assign(h_wire_vars + (NW - 1) * n, h_wire_vars + (NW - 1) * n + num_inputs);
    }
    B200_LAUNCH(k_sigma_evals, grid_for(NW * n, 256), 256, 0, st)(d_perm, pk->dom, n, pk->k, pk->sig_evals);
    cudaMemcpyAsync(pk->sig_coeffs, pk->sig_evals, NW * n * sizeof(fe), cudaMemcpyDeviceToDevice, st);
    if ((rc = ntt_device(dn, pk->sig_coeffs, scratch, 1, 0, NW, n, st)) != B200_OK) return fail(rc);
    // resident evaluations of the 18 fixed polynomials on the quotient domain
    if ((rc = coset_evals(pk, dn, pk->sel_coeffs, n, n, NS, pk->ce_sel, scratch, st)) != B200_OK) return fail(rc);
    if ((rc = coset_evals(pk, dn, pk->sig_coeffs, n, n, NW, pk->ce_sig, scratch, st)) != B200_OK) return fail(rc);
    if (cudaStreamSynchronize(st) != cudaSuccess) return fail(cuda_fail(cudaGetLastError(), "preprocess"));
    cudaFree(d_perm);
    d_perm = nullptr;
    // the 18 commitments of the verifying key
    if ((rc = commit_batch(c, pk, pk->sel_coeffs, n, n, NS, pk->sel_comms)) != B200_OK) return fail(rc);
    if ((rc = commit_batch(c, pk, pk->sig_coeffs, n, n, NW, pk->sig_comms)) != B200_OK) return fail(rc);
    *out = pk;
    return B200_OK;
}

struct ProofOut {  // same field order and layout as b200_proof / PlonkProofDef
    g1_affine wires_poly_comms[NW];
    g1_affine prod_perm_poly_comm;
    g1_affine split_quot_poly_comms[NW];
    g1_affine opening_proof;
    g1_affine shifted_opening_proof;
    fe wires_evals[NW];
    fe wire_sigma_evals[NW - 1];
    fe perm_next_eval;
};
static_assert(sizeof(ProofOut) == sizeof(b200_proof), "proof layout");

// ---- prover rounds as CUDA graphs ---------------------------------------------------------------
// The launches of a proof depend on (context, key) only — every per-proof value travels through ProofParams — so each
// segment between two host synchronisations is captured once (second proof of a key on a context; the first runs
// eagerly and sizes every buffer) and replayed as ONE submission afterwards: ~90 kernel launches per proof become 7
// graph launches.  Same kernels, same order, same bytes out.
// the addresses a captured segment refers to besides the key's: every grow-only buffer of the context
static uint64_t buffer_fingerprint(const Context* c) {
    const MsmScratch& m = c->msm;
    const void* ps[] = {c->plonk_ws.p, c->ntt_scratch.p, c->ntt_scratch2.p, c->h_small.p, c->h_params.p, c->d_params.p,
                        m.counts.p, m.offsets.p, m.cursor.p, m.entries.p, m.buckets.p, m.window_sums.p, m.scalars.p,
                        m.seg_offsets.p, m.seg_bucket.p, m.seg_sums.p, m.heavy.p, m.seg_order.p, m.scan_state.p, m.tree.p,
                        m.bit_sums.p, m.h_sums.p};
    uint64_t h = 1469598103934665603ull;
    for (const void* p : ps) {
        h ^= (uint64_t)(uintptr_t)p;
        h *= 1099511628211ull;
    }
    return h;
}

static ProofGraphSet* graph_set_for(Context* c, uint64_t key, const uint64_t* sub = nullptr) {
    int on = c->use_graphs;
    if (on < 0) {
        static const bool env_on = [] {
            const char* e = std::getenv("B200_GRAPHS");
            return !(e && e[0] == '0');
        }();
        on = env_on ? 1 : 0;
    }
    if (!on) return nullptr;
    ProofGraphSet* gs = nullptr;
    const uint64_t no_sub[6] = {};
    if (!sub) sub = no_sub;
    for (ProofGraphSet* g : c->graph_sets)
        if (g->key == key && std::memcmp(g->sub, sub, sizeof(g->sub)) == 0) gs = g;
    if (!gs) {
        if (c->graph_sets.size() >= 32) {  // keys come and go: drop the least recently used set
            size_t lru = 0;
            for (size_t i = 1; i < c->graph_sets.size(); ++i)
                if (c->graph_sets[i]->last_use < c->graph_sets[lru]->last_use) lru = i;
            delete c->graph_sets[lru];
            c->graph_sets.erase(c->graph_sets.begin() + (long)lru);
        }
        gs = new ProofGraphSet();
        gs->key = key;
        std::memcpy(gs->sub, sub, sizeof(gs->sub));
        c->graph_sets.push_back(gs);
    }
    gs->last_use = ++c->graph_clock;
    const uint64_t buffers = buffer_fingerprint(c);
    if (gs->buffers != buffers || gs->timing != c->msm.timing) {  // a buffer moved since the capture (a larger key grew
                                                                  // it), or the MSM timing events were switched
        gs->timing = c->msm.timing;
        for (auto& e : gs->exec)
            if (e) {
                cudaGraphExecDestroy(e);
                e = nullptr;
            }
        gs->buffers = buffers;
    }
    return gs;
}

// Runs `fn` (which only enqueues work on `st` and on streams it forks from / joins back to `st`): directly when `gs`
// is null, else through the segment's graph, capturing it first if need be.
template <class F>
static int run_segment(ProofGraphSet* gs, int idx, cudaStream_t st, F&& fn) {
    if (!gs) return fn();
    if (!gs->exec[idx]) {
        const uint64_t k0 = t_kernel_launches;
        cudaError_t e = cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal);
        if (e != cudaSuccess) return cuda_fail(e, "cudaStreamBeginCapture");
        const int rc = fn();
        cudaGraph_t graph = nullptr;
        e = cudaStreamEndCapture(st, &graph);
        if (rc != B200_OK || e != cudaSuccess) {
            if (graph) cudaGraphDestroy(graph);
            return rc != B200_OK ? rc : cuda_fail(e, "cudaStreamEndCapture");
        }
        e = cudaGraphInstantiate(&gs->exec[idx], graph, 0);
        cudaGraphDestroy(graph);
        if (e != cudaSuccess) {
            gs->exec[idx] = nullptr;
            return cuda_fail(e, "cudaGraphInstantiate");
        }
        gs->kernels[idx] = t_kernel_launches - k0;
    } else {
        g_kernel_launches.fetch_add(gs->kernels[idx], std::memory_order_relaxed);  // the kernels this submission runs
    }
    const auto t0 = std::chrono::steady_clock::now();
    const cudaError_t e = cudaGraphLaunch(gs->exec[idx], st);
    g_launch_host_ns.fetch_add(
        (uint64_t)std::chrono::duration_cast<std::chrono::nanoseconds>(std::chrono::steady_clock::now() - t0).count(),
        std::memory_order_relaxed);
    g_graph_launches.fetch_add(1, std::memory_order_relaxed);
    if (e != cudaSuccess) return cuda_fail(e, "cudaGraphLaunch");
    return B200_OK;
}

// Commitment epilogue of a batch: from this many commitments in one MSM on, the last step of every window sum (sum_b 2^b
// T_b) runs on the device (msm_horner_kernel, one warp per window, all windows at once) instead of on the host
// (msm_finish_batch, serial in the number of commitments).  Measured with tools/prove_batch_bench.py on an H100 80GB HBM3
// at 700 W (DESIGN §6): even at 5 commitments of 2^12-2^14 points, the device ahead from 10 on (2^13: 0.64 vs 0.71 ms
// at 10, 2.85 vs 3.86 ms at 64).
constexpr unsigned kDeviceHornerFrom = 10;

// Enqueue `count` commitments as segment `idx` (after `before`'s launches); `*pending` is the batch for commit_collect.
template <class F>
static int commit_enqueue(Context* c, MsmScratch* msm, const Bases* srs, ProofGraphSet* gs, bool single, int idx, const fe* d_coeffs,
                          size_t len, size_t stride, unsigned count, MsmPending* pending, F&& before) {
    cudaStream_t st = c->stream;
    const MsmEpilogue e = single || count < kDeviceHornerFrom ? MsmEpilogue::HostBits : MsmEpilogue::HostWindows;
    const int r = run_segment(gs, idx, st, [&]() -> int {
        const int r2 = before();
        if (r2 != B200_OK) return r2;
        return msm_launch_batch(srs, 0, d_coeffs, len, stride, count, /*montgomery=*/1, e, msm, st, pending);
    });
    if (r != B200_OK) return r;
    if (gs) {  // a graph launch: the batch the captured launch describes, and the event it leaves to its caller
        *pending = msm_pending(srs, len, count, e);
        B200_CUDA(cudaEventRecord(msm->done_ev, st));
    }
    return B200_OK;
}

static int commit_collect(MsmScratch* msm, const MsmPending& pending, g1_affine* out) {
    std::vector<int> inf(pending.batch);
    const int rc = msm_finish_batch(msm, pending, out, inf.data());
    if (rc != B200_OK) return rc;
    for (unsigned i = 0; i < pending.batch; ++i)
        if (inf[i]) std::memset(&out[i], 0, sizeof(out[i]));
    return B200_OK;
}

static void fill_open_params(OpenParams* o, fe z) {
    for (int l = 0; l < kLevels; ++l) {
        o->z[l] = z;
        o->zp[l].v[0] = fe_one<Fr>();
        for (int e = 1; e <= CH; ++e) o->zp[l].v[e] = FMUL(o->zp[l].v[e - 1], z);
        z = o->zp[l].v[CH];
    }
}

// One proof of a prover call: its inputs, its outputs, and its status (B200_OK, or B200_ERR_UNSATISFIED when the witness
// does not satisfy the circuit).
struct ProveItem {
    const fe* wires;       // the 5 x n table, or null: the table is gathered from `witness` through the key's wiring
    const fe* pub_inputs;  // with a witness: filled in by prove()
    const fe* blinders;
    ProofOut* proof;
    fe* link_poly;
    fe* challenges;
    int status;
    const fe* witness = nullptr;   // num_vars elements, host or device pointer
    fe* pub_inputs_out = nullptr;  // with a witness, may be null: receives the public inputs
};

// A pointer the device can read in place (cudaMalloc'ed or managed memory), as opposed to host memory
static bool device_readable(const void* p) {
    cudaPointerAttributes a;
    if (cudaPointerGetAttributes(&a, p) != cudaSuccess) {
        cudaGetLastError();
        return false;
    }
    return a.type == cudaMemoryTypeDevice || a.type == cudaMemoryTypeManaged;
}

// The buffers a prover call runs in: the context's own (single proofs; their captured graphs refer to these addresses)
// or the context's batch set (Context::batch), which batches grow instead.
struct ProverBufs {
    DevBuf *ws, *nscr, *nscr2, *d_params;
    HostPinned *h_small, *h_params;
    MsmScratch* msm;
};
static ProverBufs single_bufs(Context* c) {
    return {&c->plonk_ws, &c->ntt_scratch, &c->ntt_scratch2, &c->d_params, &c->h_small, &c->h_params, &c->msm};
}
static ProverBufs batch_bufs(Context* c) {
    Context::BatchBufs& b = c->batch;
    return {&b.ws, &b.nscr, &b.nscr2, &b.d_params, &b.h_small, &b.h_params, &b.msm};
}

// The value at zeta that the verifier expects of the batched polynomial opened at zeta (lin + sum v^i w_i + sum
// v^(5+i) sigma_i): E = -r0 + sum v^i w_i(zeta) + sum v^(5+i) sigma_i(zeta), read from vt::plonk_terms (with u = 0 the
// generator's B scalar is -E).  The proof verifies only if the polynomial takes this value at zeta; for a witness that
// satisfies the circuit it does.  The 1 / (n (zeta - w^j)) of the public inputs come from one batch inversion.
static fe expected_opening(const ProvingKey* pk, const fe* pub, const ProofOut& proof, const fe ch[5]) {
    const size_t cnt = std::max<size_t>(pk->num_inputs, 1);  // j = 0 also gives L_1's denominator
    std::vector<fe> wpow(cnt), inv(cnt);
    const fe nfr = host_from_u64(pk->n);
    fe acc = fe_one<Fr>(), wj = fe_one<Fr>();
    for (size_t j = 0; j < cnt; ++j) {  // inv[j]: the product of the denominators before j
        wpow[j] = wj;
        inv[j] = acc;
        acc = FMUL(acc, FMUL(FSUB(ch[3], wj), nfr));
        wj = FMUL(wj, pk->group_gen);
    }
    acc = fe_inv<Fr>(acc);
    for (size_t j = cnt; j-- > 0;) {
        const fe d = FMUL(FSUB(ch[3], wpow[j]), nfr);
        inv[j] = FMUL(inv[j], acc);
        acc = FMUL(acc, d);
    }
    struct Den {
        const fe *inv, *wpow;
        void get(size_t j, fe* i, fe* w) const {
            *i = inv[j];
            *w = wpow[j];
        }
    } den{inv.data(), wpow.data()};
    struct Sink {
        fe g = fe_zero();
        void operator()(int slot, int side, const fe& s) {
            if (slot == vt::kSlotG && side == vt::kSideB) g = s;
        }
    } sink;
    const vt::PlonkChallenges pc{ch[0], ch[1], ch[2], ch[3], ch[4], fe_zero()};
    vt::plonk_terms(pk->log_n, pk->num_inputs, pk->k.v, pub, *reinterpret_cast<const vt::ProofIn*>(&proof), pc,
                    pk->group_gen, den, sink);
    return fe_neg<Fr>(sink.g);
}

// The five prover rounds for k proofs of one key.  Every launch covers all k proofs (see Workspace and the kernels'
// batch index); every commitment round is ONE batched MSM over the k proofs' polynomials; the host runs the k
// Fiat–Shamir transcripts between rounds, so a batch makes the five host round trips once.
// single: b200_plonk_prove (k = 1 on the context's own buffers, each segment replayed as a CUDA graph from the second
// proof of a key on); otherwise a batch, eager, on Context::batch.  An unsatisfied item gets B200_ERR_UNSATISFIED in its
// status and incomplete outputs; the others are proved.  When no item is left after round 3 the call returns
// B200_ERR_UNSATISFIED.
static int prove(Context* c, const ProverBufs& bf, const ProvingKey* pk, ProveItem* items, unsigned k, bool single) {
    const size_t n = pk->n, m = pk->m;
    const unsigned log_n = pk->log_n;
    cudaStream_t st = c->stream;
    int rc;
    // h_small: the k degree flags, then k x 2 NW evaluations, then the k batched polynomials' values at zeta
    const size_t flags_bytes = ((size_t)k * 4 + 63) / 64 * 64;
    if ((rc = bf.ws->reserve(workspace_elems(n, k) * sizeof(fe))) != B200_OK) return rc;
    const bool from_witness = items[0].witness != nullptr;  // every item of a call has the same kind of input
    // the NTT scratch doubles as the staging area of the witness vectors: the gather has read them before round 1 uses it
    if ((rc = bf.nscr->reserve((size_t)k * std::max(7 * m, from_witness ? pk->num_vars : 0) * sizeof(fe))) != B200_OK) return rc;
    if ((rc = bf.nscr2->reserve((size_t)k * 6 * m * sizeof(fe))) != B200_OK) return rc;
    if ((rc = bf.h_small->reserve(std::max<size_t>(4096, flags_bytes + (size_t)k * (2 * NW + 1) * sizeof(fe)))) != B200_OK) return rc;
    if ((rc = bf.h_params->reserve(k * sizeof(ProofParams))) != B200_OK) return rc;
    if ((rc = bf.d_params->reserve(k * sizeof(ProofParams))) != B200_OK) return rc;
    if (!c->stream2) {
        B200_CUDA(cudaStreamCreateWithPriority(&c->stream2, cudaStreamNonBlocking, c->stream2_prio));
        B200_CUDA(cudaEventCreateWithFlags(&c->ev_fork, cudaEventDisableTiming));
        B200_CUDA(cudaEventCreateWithFlags(&c->ev_join, cudaEventDisableTiming));
    }
    Workspace w = carve(reinterpret_cast<fe*>(bf.ws->p), n, k);
    fe* nscr = reinterpret_cast<fe*>(bf.nscr->p);
    const size_t S = w.S;
    Domain* dn = nullptr;
    if ((rc = get_domain(c, log_n, &dn)) != B200_OK) return rc;
    const fe one = fe_one<Fr>();

    // graphs: only once a proof of this key has run eagerly on this context (every buffer has its final size then)
    ProofGraphSet* gset = single ? graph_set_for(c, pk->id) : nullptr;
    ProofGraphSet* gs = gset && gset->proofs_seen > 0 ? gset : nullptr;
    ProofParams* hp = reinterpret_cast<ProofParams*>(bf.h_params->p);  // pinned staging copy, one block per proof
    ProofParams* dp = reinterpret_cast<ProofParams*>(bf.d_params->p);  // what the kernels read
    static_assert(sizeof(ProofParams) % sizeof(fe) == 0, "ProofParams is an array of field elements");
    constexpr size_t D = sizeof(ProofParams) / sizeof(fe);  // elements from one proof's parameters to the next's
    // first operation of every segment that follows a host update of hp[]
    auto push_params = [&]() -> int {
        B200_CUDA(cudaMemcpyAsync(dp, hp, k * sizeof(ProofParams), cudaMemcpyHostToDevice, st));
        return B200_OK;
    };
    MsmPending pending;  // the commitments between commit_enqueue and commit_collect
    auto commit_enqueue = [&](int idx, const fe* d_coeffs, size_t len, size_t stride, unsigned count, auto&& before) -> int {
        return b200::commit_enqueue(c, bf.msm, pk->srs, gs, single, idx, d_coeffs, len, stride, count, &pending, before);
    };
    auto nothing = []() -> int { return B200_OK; };
    std::vector<g1_affine> comms((size_t)NW * k);  // the commitments of the current round, [proof][i]

    using clk = std::chrono::steady_clock;
    auto t_prev = clk::now();
    int phase = 0;
    auto mark = [&]() {  // wall time between sync points (every commit synchronises the stream)
        const auto now = clk::now();
        if (phase < 8) c->plonk_ms[phase++] = std::chrono::duration<float, std::milli>(now - t_prev).count();
        t_prev = now;
    };
    // ---- inputs -------------------------------------------------------------------------------------
    // caller-owned buffers are copied outside the graphs (their addresses change from proof to proof)
    B200_CUDA(cudaMemsetAsync(w.wpoly, 0, (NW + 1) * k * S * sizeof(fe), st));  // wire slots and the public-input slots behind them
    std::vector<fe> pubs;  // the public inputs of witness items
    if (from_witness) {
        const size_t nv = pk->num_vars, ni = pk->num_inputs;
        pubs.resize((size_t)k * ni);
        bool any_device = false;
        for (unsigned p0 = 0; p0 < k; p0 += kMaxBatchChunk) {
            const unsigned cnt = std::min<unsigned>(k - p0, kMaxBatchChunk);
            WitnessPtrs wit{};
            for (unsigned q = 0; q < cnt; ++q) {
                const unsigned p = p0 + q;
                const bool in_place = device_readable(items[p].witness) && (uintptr_t)items[p].witness % alignof(fe) == 0;
                if (in_place) {
                    wit.v[q] = items[p].witness;
                } else {  // host memory (or a device pointer the 16-byte loads cannot take): staged
                    fe* stage = nscr + (size_t)p * nv;
                    B200_CUDA(cudaMemcpyAsync(stage, items[p].witness, nv * sizeof(fe), cudaMemcpyDefault, st));
                    wit.v[q] = stage;
                }
                fe* pub = pubs.data() + (size_t)p * ni;
                if (!device_readable(items[p].witness)) {
                    for (size_t i = 0; i < ni; ++i) pub[i] = items[p].witness[pk->pub_vars[i]];
                } else if (ni) {
                    any_device = true;
                }
            }
            B200_LAUNCH(k_gather_wires, dim3(grid_for(NW * n, 256), cnt), 256, 0, st)(
                pk->wire_vars, wit, n, ni, w.wires_ev + (size_t)p0 * NW * n, w.pi_poly + (size_t)p0 * S, S);
        }
        if (any_device) {  // the transcript starts with the public inputs: one read-back and wait for device witnesses
            for (unsigned p = 0; p < k; ++p)
                if (device_readable(items[p].witness))
                    B200_CUDA(cudaMemcpyAsync(pubs.data() + (size_t)p * ni, w.pi_poly + (size_t)p * S, ni * sizeof(fe),
                                              cudaMemcpyDeviceToHost, st));
            B200_CUDA(cudaStreamSynchronize(st));
        }
        for (unsigned p = 0; p < k; ++p) {
            items[p].pub_inputs = pubs.data() + (size_t)p * ni;
            if (items[p].pub_inputs_out && ni) std::memcpy(items[p].pub_inputs_out, items[p].pub_inputs, ni * sizeof(fe));
        }
    } else {
        for (unsigned p = 0; p < k; ++p)  // host or device pointer (UVA)
            B200_CUDA(cudaMemcpyAsync(w.wires_ev + (size_t)p * NW * n, items[p].wires, NW * n * sizeof(fe), cudaMemcpyDefault, st));
        if (pk->num_inputs)
            for (unsigned p = 0; p < k; ++p)
                B200_CUDA(cudaMemcpyAsync(w.pi_poly + (size_t)p * S, items[p].pub_inputs, pk->num_inputs * sizeof(fe),
                                          cudaMemcpyHostToDevice, st));
    }
    std::vector<SolidityTranscript> trs(k);
    for (unsigned p = 0; p < k; ++p) {
        items[p].status = B200_OK;
        SolidityTranscript& tr = trs[p];
        tr.append_u32_be(254);  // field size in bits
        tr.append_u64_be((uint64_t)n);
        tr.append_u64_be((uint64_t)pk->num_inputs);
        for (int i = 0; i < NW; ++i) tr.append_field_elem(pk->k.v[i]);
        for (int s = 0; s < NS; ++s) tr.append_commitment(pk->sel_comms[s]);
        for (int i = 0; i < NW; ++i) tr.append_commitment(pk->sig_comms[i]);
        for (size_t i = 0; i < pk->num_inputs; ++i) tr.append_field_elem(items[p].pub_inputs[i]);
    }

    // ---- round 1 ------------------------------------------------------------------------------------
    for (unsigned p = 0; p < k; ++p)
        for (int i = 0; i < NW; ++i) {
            hp[p].blind_w[i][0] = items[p].blinders[2 * i];
            hp[p].blind_w[i][1] = items[p].blinders[2 * i + 1];
        }
    rc = run_segment(gs, 0, st, [&]() -> int {
        int r = push_params();
        if (r != B200_OK) return r;
        B200_CUDA(cudaMemcpy2DAsync(w.wpoly, S * sizeof(fe), w.wires_ev, n * sizeof(fe), n * sizeof(fe), NW * k,
                                    cudaMemcpyDeviceToDevice, st));
        {
            // wires and public inputs: evaluations -> coefficients, one batch of 6k (pi_poly sits directly behind wpoly)
            HeavyScope hv(c, st);
            if ((r = ntt_device(dn, w.wpoly, nscr, 1, 0, (NW + 1) * k, S, hv.run)) != B200_OK) return r;
        }
        B200_LAUNCH(k_blind_wires, k, 32, 0, st)(w.wpoly, S, n, &dp->blind_w[0][0], D);
        return B200_OK;
    });
    if (rc != B200_OK) return rc;
    // Fork: the coset evaluations of the 5 wire polynomials and of the public-input polynomial do not
    // depend on any challenge, so they run on a second stream underneath the round-1/2 commitments
    // (whose bucket reduction and host round trip leave most SMs idle).
    struct Side {
        Context* c;
        bool pending = false;
        ~Side() {
            if (pending) cudaStreamSynchronize(c->stream2);  // error paths: never leave the side stream running
        }
    } side{c};
    {
        cudaStream_t s2 = c->stream2;
        B200_CUDA(cudaEventRecord(c->ev_fork, st));
        B200_CUDA(cudaStreamWaitEvent(s2, c->ev_fork, 0));
        side.pending = true;
        // 5k wire polynomials (n + 2 coefficients) and the k public-input polynomials (n, zero tail) in one batch
        rc = run_segment(gs, 1, s2, [&]() -> int {
            return coset_evals(pk, dn, w.wpoly, S, n + 2, (NW + 1) * k, w.ext, reinterpret_cast<fe*>(bf.nscr2->p), s2);
        });
        if (rc != B200_OK) return rc;
        B200_CUDA(cudaEventRecord(c->ev_join, s2));
    }
    if ((rc = commit_enqueue(2, w.wpoly, n + 2, S, NW * k, nothing)) != B200_OK) return rc;
    if ((rc = commit_collect(bf.msm, pending, comms.data())) != B200_OK) return rc;
    for (unsigned p = 0; p < k; ++p) {
        ProofOut* proof = items[p].proof;
        std::memcpy(proof->wires_poly_comms, &comms[(size_t)p * NW], sizeof(proof->wires_poly_comms));
        if (items[p].link_poly)  // completes under round 2; the stream is synchronised several times before this call returns
            B200_CUDA(cudaMemcpyAsync(items[p].link_poly, w.wpoly + (size_t)p * NW * S, (n + 2) * sizeof(fe), cudaMemcpyDeviceToHost, st));
        for (int i = 0; i < NW; ++i) trs[p].append_commitment(proof->wires_poly_comms[i]);
    }
    mark();  // [0] round 1

    // ---- round 2 ------------------------------------------------------------------------------------
    std::vector<fe> beta(k), gamma(k), alpha(k), zeta(k), zeta_w(k), v(k);
    for (unsigned p = 0; p < k; ++p) {
        beta[p] = trs[p].get_and_append_challenge();
        gamma[p] = trs[p].get_and_append_challenge();
        hp[p].chal[0] = beta[p];
        hp[p].chal[1] = gamma[p];
        for (int i = 0; i < 3; ++i) hp[p].blind_z[i] = items[p].blinders[10 + i];
    }
    rc = commit_enqueue(3, w.zpoly, n + 3, S, k, [&]() -> int {
        int r = push_params();
        if (r != B200_OK) return r;
        B200_LAUNCH(k_perm_num_den, dim3(grid_for(n, 128), k), 128, 0, st)(w.wires_ev, pk->sig_evals, pk->dom, pk->k, &dp->chal[0], D, n,
                                                                           w.num, w.den);
        batch_inverse_enqueue(w.num, w.den, w.tmp, k * n, st);  // the k proofs' denominators as one vector
        scan_mul_exclusive(w.den, n, k, w.scan, st);             // z(w^j) = prod_{i<j} ratio_i, per proof
        B200_CUDA(cudaMemsetAsync(w.zpoly, 0, k * S * sizeof(fe), st));
        B200_CUDA(cudaMemcpy2DAsync(w.zpoly, S * sizeof(fe), w.den, n * sizeof(fe), n * sizeof(fe), k, cudaMemcpyDeviceToDevice, st));
        if ((r = ntt_device(dn, w.zpoly, nscr, 1, 0, k, S, st)) != B200_OK) return r;
        BlindArgs b{};
        b.count = 3;
        b.dyn = &dp->blind_z[0];
        B200_LAUNCH(k_blind, k, 32, 0, st)(w.zpoly, n, b, S, D);
        return B200_OK;
    });
    if (rc != B200_OK) return rc;
    if ((rc = commit_collect(bf.msm, pending, comms.data())) != B200_OK) return rc;
    for (unsigned p = 0; p < k; ++p) {
        items[p].proof->prod_perm_poly_comm = comms[p];
        trs[p].append_commitment(comms[p]);
    }
    mark();  // [1] round 2

    // ---- round 3 ------------------------------------------------------------------------------------
    for (unsigned p = 0; p < k; ++p) {
        alpha[p] = trs[p].get_and_append_challenge();
        hp[p].chal[2] = alpha[p];
        hp[p].chal[3] = fe_sqr<Fr>(alpha[p]);
        for (int i = 0; i < 4; ++i) hp[p].blind_q[i] = items[p].blinders[13 + i];
    }
    B200_CUDA(cudaStreamWaitEvent(st, c->ev_join, 0));  // join: wire / PI coset evaluations are ready
    side.pending = false;
    const size_t deg = NW * (n + 1) + 2;
    uint32_t* h_flag = reinterpret_cast<uint32_t*>(bf.h_small->p);  // pinned; read after the commitments below are in
    mark();  // [2] round 3 (host part)
    // the last chunk has n coefficients; its tail up to n + 3 is zero, so one batch length serves
    rc = commit_enqueue(4, w.split, n + 3, S, NW * k, [&]() -> int {
        int r = push_params();
        if (r != B200_OK) return r;
        {
            HeavyScope hv(c, st);
            if ((r = coset_evals(pk, dn, w.zpoly, S, n + 3, k, w.zext, nscr, hv.run)) != B200_OK) return r;
        }
        {
            QuotArgs q;
            q.sel = pk->ce_sel;
            q.sig = pk->ce_sig;
            q.ext = w.ext;
            q.pi = w.ext + (size_t)k * NW * m;  // the public-input evaluations follow all k proofs' wire evaluations
            q.zext = w.zext;
            q.pts = pk->coset_pts;
            q.l1_inv = pk->l1_inv;
            q.out = w.quot;
            q.m = m;
            q.log_n = log_n;
            q.k = pk->k;
            q.chal = &dp->chal[0];
            q.dstride = D;
            for (int i = 0; i < 8; ++i) q.zh_inv[i] = pk->zh_inv[i];
            HeavyScope hv(c, st);
            B200_LAUNCH(k_quotient, dim3(grid_for(m, 128), k), 128, 0, hv.run)(q);
            // back to coefficients: nc size-n inverse transforms per proof, then un-scale and un-mix the cosets
            if ((r = ntt_device(dn, w.quot, nscr, 1, 0, (unsigned)pk->nc * k, n, hv.run)) != B200_OK) return r;
            if (pk->nc == 6) B200_LAUNCH(k_coset_combine<6>, dim3(grid_for(n, 128), k), 128, 0, hv.run)(w.quot, n, pk->cscale_inv, pk->comb);
            else B200_LAUNCH(k_coset_combine<8>, dim3(grid_for(n, 128), k), 128, 0, hv.run)(w.quot, n, pk->cscale_inv, pk->comb);
        }
        B200_CUDA(cudaMemsetAsync(w.flag, 0, 4 * k, st));
        B200_LAUNCH(k_check_degree, dim3(grid_for(m - deg, 256), k), 256, 0, st)(w.quot, deg, m, w.flag);
        B200_CUDA(cudaMemcpyAsync(h_flag, w.flag, 4 * k, cudaMemcpyDeviceToHost, st));
        B200_LAUNCH(k_split_quotient, dim3(grid_for(n + 3, 256), NW, k), 256, 0, st)(w.quot, m, n, S, &dp->blind_q[0], D, w.split);
        return B200_OK;
    });
    if (rc != B200_OK) return rc;
    if ((rc = commit_collect(bf.msm, pending, comms.data())) != B200_OK) return rc;
    unsigned satisfied = 0;
    for (unsigned p = 0; p < k; ++p) {  // the flags were copied before the commitments' window sums on the same stream
        if (h_flag[p]) items[p].status = B200_ERR_UNSATISFIED;
        else ++satisfied;
    }
    if (!satisfied) {
        set_error("WrongQuotientPolyDegree: the witness does not satisfy the circuit");
        return B200_ERR_UNSATISFIED;
    }
    for (unsigned p = 0; p < k; ++p) {
        ProofOut* proof = items[p].proof;
        std::memcpy(proof->split_quot_poly_comms, &comms[(size_t)p * NW], sizeof(proof->split_quot_poly_comms));
        for (int i = 0; i < NW; ++i) trs[p].append_commitment(proof->split_quot_poly_comms[i]);
    }
    mark();  // [3] round 3: quotient and its 5 commitments

    // ---- round 4 ------------------------------------------------------------------------------------
    for (unsigned p = 0; p < k; ++p) {
        zeta[p] = trs[p].get_and_append_challenge();
        zeta_w[p] = FMUL(zeta[p], pk->group_gen);
    }
    fe* h_evals = reinterpret_cast<fe*>(reinterpret_cast<char*>(bf.h_small->p) + flags_bytes);  // pinned, [proof][2 NW]
    fe* h_bz = h_evals + (size_t)k * 2 * NW;                                                      // pinned, [proof]
    {
        // proof 0's polynomials; proof p's are `pstrides` further (the key's sigmas are shared)
        const fe* polys[kMaxEval];
        size_t lens[kMaxEval], pstrides[kMaxEval];
        for (int i = 0; i < NW; ++i) { polys[i] = w.wpoly + (size_t)i * S; lens[i] = n + 2; pstrides[i] = NW * S; }
        for (int i = 0; i < NW - 1; ++i) { polys[NW + i] = pk->sig_coeffs + (size_t)i * n; lens[NW + i] = n; pstrides[NW + i] = 0; }
        polys[2 * NW - 1] = w.zpoly; lens[2 * NW - 1] = n + 3; pstrides[2 * NW - 1] = S;
        for (unsigned p = 0; p < k; ++p)
            for (int q = 0; q < 2 * NW; ++q) {
                fe z = q == 2 * NW - 1 ? zeta_w[p] : zeta[p];
                for (int l = 0; l < kLevels; ++l) {
                    hp[p].eval_z[l][q] = z;
                    z = host_pow(z, CH);
                }
            }
        rc = run_segment(gs, 5, st, [&]() -> int {
            int r = push_params();
            if (r != B200_OK) return r;
            eval_batch(polys, lens, nullptr, 2 * NW, w.evals, w.escr, st, dp->eval_z, k, pstrides, kEvalSlots, D);
            B200_CUDA(cudaMemcpy2DAsync(h_evals, 2 * NW * sizeof(fe), w.evals, kEvalSlots * sizeof(fe), 2 * NW * sizeof(fe), k,
                                        cudaMemcpyDeviceToHost, st));
            return B200_OK;
        });
        if (rc != B200_OK) return rc;
    }
    B200_CUDA(cudaStreamSynchronize(st));
    for (unsigned p = 0; p < k; ++p) {
        ProofOut* proof = items[p].proof;
        const fe* he = h_evals + (size_t)p * 2 * NW;
        for (int i = 0; i < NW; ++i) proof->wires_evals[i] = he[i];
        for (int i = 0; i < NW - 1; ++i) proof->wire_sigma_evals[i] = he[NW + i];
        proof->perm_next_eval = he[2 * NW - 1];
        for (int i = 0; i < NW; ++i) trs[p].append_field_elem(proof->wires_evals[i]);
        for (int i = 0; i < NW - 1; ++i) trs[p].append_field_elem(proof->wire_sigma_evals[i]);
        trs[p].append_field_elem(proof->perm_next_eval);
    }
    mark();  // [4] round 4

    // ---- round 5 ------------------------------------------------------------------------------------
    // pointers and lengths (proof 0's, and the stride to proof p's): launch arguments; scalars: ProofParams
    LinArgs la{};
    for (unsigned p = 0; p < k; ++p) {
        v[p] = trs[p].get_and_append_challenge();
        const ProofOut* proof = items[p].proof;
        const fe* we = proof->wires_evals;
        const fe* se = proof->wire_sigma_evals;
        const fe al = alpha[p], be = beta[p], ga = gamma[p], ze = zeta[p];
        int t = 0;
        auto push = [&](const fe* ptr, size_t pstride, size_t len, const fe& s) {
            la.p[t] = ptr;
            la.pstride[t] = (uint32_t)pstride;
            la.len[t] = (uint32_t)len;
            hp[p].lin_s[t] = s;
            ++t;
        };
        auto pow5 = [&](const fe& x) { return FMUL(fe_sqr<Fr>(fe_sqr<Fr>(x)), x); };
        const fe* sel = pk->sel_coeffs;
        for (int j = 0; j < 4; ++j) push(sel + (size_t)j * n, 0, n, we[j]);
        push(sel + 4 * n, 0, n, FMUL(we[0], we[1]));
        push(sel + 5 * n, 0, n, FMUL(we[2], we[3]));
        for (int j = 0; j < 4; ++j) push(sel + (size_t)(6 + j) * n, 0, n, pow5(we[j]));
        push(sel + 10 * n, 0, n, fe_neg<Fr>(we[4]));
        push(sel + 11 * n, 0, n, one);
        push(sel + 12 * n, 0, n, FMUL(FMUL(FMUL(we[0], we[1]), FMUL(we[2], we[3])), we[4]));
        // z(X): alpha prod(w_i + beta k_i zeta + gamma) + alpha^2 L1(zeta)
        const fe vanish = FSUB(host_pow(ze, n), one);
        const fe l1 = FMUL(vanish, fe_inv<Fr>(FMUL(host_from_u64(n), FSUB(ze, one))));
        fe cz = al;
        for (int j = 0; j < NW; ++j) cz = FMUL(cz, FADD(FADD(we[j], FMUL(FMUL(pk->k.v[j], ze), be)), ga));
        cz = FADD(cz, FMUL(fe_sqr<Fr>(al), l1));
        push(w.zpoly, S, n + 3, cz);
        // sigma_4(X): -alpha beta z(zeta w) prod_{i<4}(w_i + beta sigma_i + gamma)
        fe cs = FMUL(FMUL(al, be), proof->perm_next_eval);
        for (int j = 0; j < NW - 1; ++j) cs = FMUL(cs, FADD(FADD(we[j], FMUL(be, se[j])), ga));
        push(pk->sig_coeffs + (size_t)(NW - 1) * n, 0, n, fe_neg<Fr>(cs));
        // - Z_H(zeta) * sum zeta^((n+2) i) t_i(X)
        const fe zn2 = FMUL(FMUL(FADD(vanish, one), ze), ze);
        fe ct = fe_neg<Fr>(vanish);
        for (int i = 0; i < NW; ++i) {
            push(w.split + (size_t)i * S, NW * S, i < NW - 1 ? n + 3 : n, ct);
            ct = FMUL(ct, zn2);
        }
        // batched opening at zeta: lin + v w_0 + ... + v^5 w_4 + v^6 sigma_0 + ... + v^9 sigma_3
        fe cv = one;
        for (int i = 0; i < NW; ++i) {
            cv = FMUL(cv, v[p]);
            push(w.wpoly + (size_t)i * S, NW * S, n + 2, cv);
        }
        for (int i = 0; i < NW - 1; ++i) {
            cv = FMUL(cv, v[p]);
            push(pk->sig_coeffs + (size_t)i * n, 0, n, cv);
        }
        la.count = t;
        fill_open_params(&hp[p].open[0], ze);
        fill_open_params(&hp[p].open[1], zeta_w[p]);
    }
    la.dyn = &dp->lin_s[0];
    la.dstride = D;
    rc = commit_enqueue(6, w.sdiv + 1, n + 2, S + 8, 2 * k, [&]() -> int {
        int r = push_params();
        if (r != B200_OK) return r;
        B200_LAUNCH(k_lincomb, dim3(grid_for(n + 3, 128), k), 128, 0, st)(la, n + 3, w.lin, S);
        // opening proofs: commit((batch - batch(zeta)) / (X - zeta)) and commit((z - z(zeta w)) / (X - zeta w))
        HornerStrides hs;
        hs.k = k;
        hs.p = S;
        hs.s = 2 * (S + 8);
        hs.out = kEvalSlots;
        hs.dyn = D;
        horner_suffix(w.lin, n + 3, zeta[0], w.sdiv, w.evals + 16, w.hscr, st, &dp->open[0], hs);
        horner_suffix(w.zpoly, n + 3, zeta_w[0], w.sdiv + (S + 8), w.evals + 17, w.hscr, st, &dp->open[1], hs);
        B200_CUDA(cudaMemcpy2DAsync(h_bz, sizeof(fe), w.evals + 16, kEvalSlots * sizeof(fe), sizeof(fe), k,
                                    cudaMemcpyDeviceToHost, st));
        return B200_OK;
    });
    if (rc != B200_OK) return rc;
    // Self-check at zeta, on the host while the opening commitments run: the batched polynomial must take the value the
    // verifier expects.  Round 3's degree check reads a quotient interpolated from 6 cosets, which misses every witness
    // whose per-row violations are the values on H of a polynomial of degree <= 7 (DESIGN §4); this check refuses those,
    // except with probability at most (6n + 8) / r.
    std::vector<fe> want_bz(k);
    {
        const auto t0 = clk::now();
        for (unsigned p = 0; p < k; ++p) {
            const fe ch[5] = {beta[p], gamma[p], alpha[p], zeta[p], v[p]};
            if (items[p].status == B200_OK) want_bz[p] = expected_opening(pk, items[p].pub_inputs, *items[p].proof, ch);
        }
        c->plonk_ms[6] = std::chrono::duration<float, std::milli>(clk::now() - t0).count();
    }
    comms.resize(2 * k);
    if ((rc = commit_collect(bf.msm, pending, comms.data())) != B200_OK) return rc;
    for (unsigned p = 0; p < k; ++p) {
        items[p].proof->opening_proof = comms[2 * p];
        items[p].proof->shifted_opening_proof = comms[2 * p + 1];
    }
    mark();  // [5] round 5
    if (gset && !gs) gset->proofs_seen = 1;  // this key has now run eagerly on this context: later proofs replay graphs
    satisfied = 0;
    for (unsigned p = 0; p < k; ++p) {  // h_bz was copied before the opening commitments on the same stream
        if (items[p].status == B200_OK && !fe_eq(h_bz[p], want_bz[p])) items[p].status = B200_ERR_UNSATISFIED;
        if (items[p].status == B200_OK) ++satisfied;
    }
    if (!satisfied) {
        set_error("WrongQuotientPolyDegree: the witness does not satisfy the circuit");
        return B200_ERR_UNSATISFIED;
    }
    for (unsigned p = 0; p < k; ++p) {
        if (!items[p].challenges || items[p].status != B200_OK) continue;
        SolidityTranscript& tr = trs[p];
        tr.append_commitment(items[p].proof->opening_proof);
        tr.append_commitment(items[p].proof->shifted_opening_proof);
        const fe u = tr.get_and_append_challenge();
        const fe all[6] = {beta[p], gamma[p], alpha[p], zeta[p], v[p], u};
        std::memcpy(items[p].challenges, all, sizeof(all));
    }
    return B200_OK;
}

// Proofs per prove() call of a batch: as many as half the free device memory holds (the batch buffers the context
// already has count as free: they are reused), at most kMaxBatchChunk.  Per proof: the workspace, the two NTT scratches
// and the MSM scratch of its five largest commitments.  B200_PROVE_BATCH_CHUNK overrides it (tests: the bytes out do
// not depend on the chunk size).
static size_t prove_batch_chunk(Context* c, const ProvingKey* pk, size_t k) {
    if (const char* e = std::getenv("B200_PROVE_BATCH_CHUNK")) {
        const long v = std::atol(e);
        if (v >= 1) return std::min<size_t>((size_t)v, k);
    }
    const size_t n = pk->n, m = pk->m;
    const MsmPlan& pl = pk->srs->plan;
    const size_t msm_per_commit = n * (size_t)pl.n_digits * 4 * 2 + ((size_t)pl.n_phys << (pl.c - 1)) * sizeof(g1_xyzz) * 4;
    // (a witness vector is staged in the first NTT scratch, 7m elements unless the vector is longer)
    const size_t per_proof = (workspace_elems(n, 1) + 6 * m + std::max(7 * m, pk->num_vars)) * sizeof(fe) + NW * msm_per_commit;
    size_t free_b = 0, total_b = 0;
    if (cudaMemGetInfo(&free_b, &total_b) != cudaSuccess) free_b = 0;
    const Context::BatchBufs& b = c->batch;
    const size_t budget = (free_b + b.ws.cap + b.nscr.cap + b.nscr2.cap) / 2;
    // the MSM's 32-bit entry index: n * digits * NW * chunk < 2^32
    const size_t idx_cap = ((size_t)1 << 32) / ((size_t)n * pl.n_digits * NW) - 1;
    return std::max<size_t>(1, std::min({k, kMaxBatchChunk, budget / per_proof, idx_cap}));
}

// ---------------------------------------------------------------------------------------------
// proof linking — replaces `PlonkKzgSnark::link_proofs::<SolidityTranscript>(hint_a, hint_b,
// &group_layout, &commit_key)` (circuits-core/src/zk_circuits/proof_linking/intent_only.rs:42-47,
// intent_and_balance.rs:66-72): q = (a1 - a2) / Z_D with Z_D = prod_{i<size} (X - g^(offset+i)),
// g the generator of the 2^alignment roots of unity (`GroupLayout`); eta from the transcript;
// opening of a1 - a2 - Z_D(eta) q at eta.  The reference divides by the `size` linear factors in turn; here the
// division runs on an evaluation domain (coset transform, pointwise division by Z_D, inverse transform): the same
// quotient, and an inexact division shows as a quotient of too high a degree.
// ---------------------------------------------------------------------------------------------
struct LinkOut {
    g1_affine quotient_commitment;
    g1_affine opening_proof;
};
static_assert(sizeof(LinkOut) == sizeof(b200_link_proof), "link proof layout");

// One link proof of a link_chunk() call: its inputs, outputs and status (B200_OK, or B200_ERR_UNSATISFIED when the
// division by Z_D is not exact).  log_N: the size of the transform its division runs on.
struct LinkItem {
    const fe *a1, *a2;
    size_t len1, len2;
    g1_affine comm1, comm2;
    unsigned alignment;
    size_t offset, size;
    LinkOut* out;
    fe* eta;
    unsigned log_N;
    int status;
};

// Checks the layout and lengths of one link proof and fills `it` from `x` (whose pointers the caller has checked):
// B200_ERR_INVALID, with a message that starts with `where`, when no link proof is made for them.
static int link_item(const Bases* srs, const b200_link_item& x, const std::string& where, LinkItem* it) {
    const size_t len = std::max(x.len1, x.len2);
    if (x.size == 0 || x.size >= len || x.alignment > 28 || len > srs->n) {
        set_error(where + ": bad group layout or polynomial length");
        return B200_ERR_INVALID;
    }
    // Division by Z_D on an evaluation domain: N = 2^log_N >= len points of the coset g * H_N (Z_D has no root there).
    // diff / Z_D pointwise, back to coefficients: the quotient when the division is exact — and exact it is iff the
    // interpolant's degree is len - 1 - size (p * Z_D - diff has degree < N and vanishes on N points).  Two transforms,
    // one batch inversion and a few element-wise kernels instead of `size` dependent synthetic divisions.
    unsigned log_N = 1;
    while (((size_t)1 << log_N) < len) ++log_N;
    if (log_N > 28) {
        set_error(where + ": polynomial too long");
        return B200_ERR_INVALID;
    }
    it->a1 = reinterpret_cast<const fe*>(x.a1);
    it->a2 = reinterpret_cast<const fe*>(x.a2);
    it->len1 = x.len1;
    it->len2 = x.len2;
    std::memcpy(&it->comm1, x.comm1, 64);
    std::memcpy(&it->comm2, x.comm2, 64);
    it->alignment = x.alignment;
    it->offset = x.offset;
    it->size = x.size;
    it->out = reinterpret_cast<LinkOut*>(x.proof);
    it->eta = reinterpret_cast<fe*>(x.eta);
    it->log_N = log_N;
    it->status = B200_OK;
    return B200_OK;
}

// Out of line: inlined into link_chunk, the transcript's std::vector::insert draws a false -Wstringop-overflow from GCC 13
__attribute__((noinline)) static fe link_eta(const g1_affine& c1, const g1_affine& c2, const g1_affine& cq) {
    SolidityTranscript tr;
    return vt::link_challenge(tr, c1, c2, cq);
}

// k link proofs at once; the items come sorted by log_N.  Each step is one launch (or one batched transform /
// inversion) over many items:
//  - the differences a1 - a2 of all k items, `L` = max len apart (zero above each item's own length);
//  - the division, per group of items of one transform size N: item y's data N apart, its roots and q_len read from its
//    LinkDesc; the quotients then go to one region `Q` = max q_len apart (zero above each item's own q_len);
//  - ONE batched MSM of the k quotients; the host runs the k transcripts (eta, Z_D(eta)) in one round trip;
//  - the openings over the common length L (leading zero coefficients change neither p(eta) nor the quotient's
//    coefficients, and zero scalars add nothing to a commitment), then ONE batched MSM of the k opening proofs.
// An item whose division is not exact is carried through the launches and gets B200_ERR_UNSATISFIED; its outputs are
// not written.
// single: b200_plonk_link (k = 1 on the context's own buffers, its two segments replayed as CUDA graphs from the second
// call with the same SRS, lengths and layout on); otherwise a batch, eager, on Context::batch.
static int link_chunk(Context* c, const ProverBufs& bf, const Bases* srs, LinkItem* const* items, unsigned k, bool single) {
    cudaStream_t st = c->stream;
    int rc;
    size_t L = 0, Q = 0, n_roots = 0, max_size = 0, max_group = 0;
    for (unsigned y = 0; y < k; ++y) {
        const LinkItem& it = *items[y];
        const size_t len = std::max(it.len1, it.len2);
        L = std::max(L, len);
        Q = std::max(Q, len - it.size);
        n_roots += it.size;
        max_size = std::max(max_size, it.size);
    }
    std::vector<unsigned> grp{0};  // group i: items [grp[i], grp[i + 1]), one transform size each
    for (unsigned y = 1; y <= k; ++y)
        if (y == k || items[y]->log_N != items[y - 1]->log_N) {
            max_group = std::max(max_group, (size_t)(y - grp.back()) << items[y - 1]->log_N);
            grp.push_back(y);
        }
    static_assert(sizeof(LinkDesc) % sizeof(fe) == 0 && sizeof(LinkParams) % sizeof(fe) == 0, "arrays of field elements");
    const size_t hscr_n = (size_t)k * 4 * (L / CH + 4 * CH + 64);
    const size_t desc_n = (size_t)k * sizeof(LinkDesc) / sizeof(fe);
    const size_t flag_n = ((size_t)k * 4 + sizeof(fe) - 1) / sizeof(fe);
    const size_t kL = (size_t)k * L, kQ = (size_t)k * Q;
    if ((rc = bf.ws->reserve((3 * kL + kQ + 3 * max_group + hscr_n + n_roots + k + desc_n + flag_n) * sizeof(fe))) != B200_OK)
        return rc;
    if ((rc = bf.nscr->reserve(max_group * sizeof(fe))) != B200_OK) return rc;
    const size_t desc_bytes = (size_t)k * sizeof(LinkDesc);
    if ((rc = bf.h_small->reserve(desc_bytes + (size_t)k * 4)) != B200_OK) return rc;
    if ((rc = bf.h_params->reserve(k * sizeof(LinkParams))) != B200_OK) return rc;
    if ((rc = bf.d_params->reserve(k * sizeof(LinkParams))) != B200_OK) return rc;
    std::vector<Domain*> doms(grp.size() - 1);
    for (size_t g = 0; g + 1 < grp.size(); ++g)
        if ((rc = get_domain(c, items[grp[g]]->log_N, &doms[g])) != B200_OK) return rc;

    fe* base = reinterpret_cast<fe*>(bf.ws->p);
    fe *d_a1 = base, *d_a2 = d_a1 + kL, *d_diff = d_a2 + kL, *d_quot = d_diff + kL;
    fe *d_E = d_quot + kQ, *d_Z = d_E + max_group, *d_ZS = d_Z + max_group;  // one group's evaluations, Z_D, scratch
    fe *hscr = d_ZS + max_group, *d_roots = hscr + hscr_n, *d_tot = d_roots + n_roots;
    LinkDesc* d_desc = reinterpret_cast<LinkDesc*>(d_tot + k);
    uint32_t* d_flag = reinterpret_cast<uint32_t*>(d_tot + k + desc_n);
    fe *d_ident = d_a1, *d_open = d_a2;  // free again once the differences are formed
    fe* nscr = reinterpret_cast<fe*>(bf.nscr->p);
    LinkDesc* h_desc = reinterpret_cast<LinkDesc*>(bf.h_small->p);
    uint32_t* h_flag = reinterpret_cast<uint32_t*>(reinterpret_cast<char*>(bf.h_small->p) + desc_bytes);
    LinkParams* hp = reinterpret_cast<LinkParams*>(bf.h_params->p);
    LinkParams* dp = reinterpret_cast<LinkParams*>(bf.d_params->p);
    constexpr size_t D = sizeof(LinkParams) / sizeof(fe);
    MsmScratch* msm = bf.msm;
    const fe one = fe_one<Fr>();

    // graphs: only once a call with this key has run eagerly on this context.  The launches depend on (context, SRS,
    // lengths, group size) only, as the layout reaches them through LinkDesc; alignment and offset stay in the key all
    // the same, so that every layout's first call runs eagerly.
    const LinkItem& i0 = *items[0];
    const uint64_t sub[6] = {srs->id, (uint64_t)i0.len1, (uint64_t)i0.len2, (uint64_t)i0.alignment, (uint64_t)i0.offset,
                             (uint64_t)i0.size};
    ProofGraphSet* gset = single ? graph_set_for(c, ~(uint64_t)0, sub) : nullptr;
    ProofGraphSet* gs = gset && gset->proofs_seen > 0 ? gset : nullptr;
    MsmPending pending;  // the commitments between commit_enqueue and commit_collect

    size_t at = 0;
    for (unsigned y = 0; y < k; ++y) {
        const LinkItem& it = *items[y];
        LinkDesc& d = h_desc[y];
        d.g = host_root_of_unity(it.alignment);
        d.root0 = host_pow(d.g, (uint64_t)it.offset);
        d.roots_at = at;
        d.size = it.size;
        d.q_len = std::max(it.len1, it.len2) - it.size;
        d.pad = 0;
        at += it.size;
    }
    // caller-owned host or device pointers (UVA) are copied outside the graphs (their addresses change from call to call)
    B200_CUDA(cudaMemsetAsync(d_a1, 0, 2 * kL * sizeof(fe), st));
    for (unsigned y = 0; y < k; ++y) {
        B200_CUDA(cudaMemcpyAsync(d_a1 + (size_t)y * L, items[y]->a1, items[y]->len1 * sizeof(fe), cudaMemcpyDefault, st));
        B200_CUDA(cudaMemcpyAsync(d_a2 + (size_t)y * L, items[y]->a2, items[y]->len2 * sizeof(fe), cudaMemcpyDefault, st));
    }
    rc = commit_enqueue(c, msm, srs, gs, single, 0, d_quot, Q, Q, k, &pending, [&]() -> int {
        int r;
        B200_CUDA(cudaMemcpyAsync(d_desc, h_desc, desc_bytes, cudaMemcpyHostToDevice, st));
        B200_CUDA(cudaMemsetAsync(d_flag, 0, (size_t)k * 4, st));
        B200_CUDA(cudaMemsetAsync(d_quot, 0, kQ * sizeof(fe), st));
        {
            LinArgs a{};
            a.count = 2;
            a.p[0] = d_a1; a.pstride[0] = (uint32_t)L; a.len[0] = (uint32_t)L; a.s[0] = one;
            a.p[1] = d_a2; a.pstride[1] = (uint32_t)L; a.len[1] = (uint32_t)L; a.s[1] = fe_neg<Fr>(one);
            B200_LAUNCH(k_lincomb, dim3(grid_for(L, 128), k), 128, 0, st)(a, L, d_diff, L);
        }
        B200_LAUNCH(k_link_roots, dim3(grid_for(max_size, 128), k), 128, 0, st)(d_desc, d_roots);
        for (size_t g = 0; g + 1 < grp.size(); ++g) {
            const unsigned y0 = grp[g], kg = grp[g + 1] - y0;
            const Domain* dN = doms[g];
            const size_t N = (size_t)1 << dN->log_n, kN = (size_t)kg * N;
            size_t min_q = N;
            for (unsigned y = y0; y < y0 + kg; ++y) min_q = std::min<size_t>(min_q, h_desc[y].q_len);
            B200_CUDA(cudaMemsetAsync(d_E, 0, kN * sizeof(fe), st));
            B200_CUDA(cudaMemcpy2DAsync(d_E, N * sizeof(fe), d_diff + (size_t)y0 * L, L * sizeof(fe), std::min(L, N) * sizeof(fe), kg,
                                        cudaMemcpyDeviceToDevice, st));
            if ((r = ntt_device(dN, d_E, nscr, /*inverse=*/0, /*coset=*/1, kg, N, st)) != B200_OK) return r;
            B200_LAUNCH(k_vanishing_on_coset_batch, dim3(grid_for(N, 128), kg), 128, 0, st)(dN->tw_fwd, N, fe_from_u32<Fr>(5), d_roots,
                                                                                            d_desc + y0, d_Z);
            batch_inverse_enqueue(nullptr, d_Z, d_ZS, kN, st);
            B200_LAUNCH(k_fr_vec_op, grid_for(kN, 256), 256, 0, st)(2, d_E, d_Z, 0, kN, d_ZS);
            if ((r = ntt_device(dN, d_ZS, nscr, /*inverse=*/1, /*coset=*/1, kg, N, st)) != B200_OK) return r;
            // a1 and a2 must agree on every root of the group, i.e. the division is exact: otherwise no link proof
            // verifies and the reference's prover output would be rejected
            B200_LAUNCH(k_check_zero_tail, dim3(grid_for(N - min_q, 256), kg), 256, 0, st)(d_ZS, N, d_desc + y0, d_flag + y0);
            // exact items are zero from q_len on, so min(Q, N) coefficients carry the whole quotient
            B200_CUDA(cudaMemcpy2DAsync(d_quot + (size_t)y0 * Q, Q * sizeof(fe), d_ZS, N * sizeof(fe), std::min(Q, N) * sizeof(fe), kg,
                                        cudaMemcpyDeviceToDevice, st));
        }
        B200_CUDA(cudaMemcpyAsync(h_flag, d_flag, (size_t)k * 4, cudaMemcpyDeviceToHost, st));
        return B200_OK;
    });
    if (rc != B200_OK) return rc;
    std::vector<g1_affine> comms(k);
    if ((rc = commit_collect(msm, pending, comms.data())) != B200_OK) return rc;
    unsigned proved = 0;
    for (unsigned y = 0; y < k; ++y) {  // the flags were copied before the commitments' window sums on the same stream
        LinkItem& it = *items[y];
        LinkParams& p = hp[y];
        std::memset(&p, 0, sizeof(p));
        if (h_flag[y]) {  // carried through the opening with harmless parameters
            it.status = B200_ERR_UNSATISFIED;
            p.lin_s[0] = one;
            fill_open_params(&p.open, fe_zero());
            continue;
        }
        ++proved;
        it.status = B200_OK;
        it.out->quotient_commitment = comms[y];
        const fe eta = link_eta(it.comm1, it.comm2, comms[y]);
        if (it.eta) *it.eta = eta;
        p.lin_s[0] = one;
        p.lin_s[1] = fe_neg<Fr>(vt::link_zd(eta, h_desc[y].g, it.offset, it.size));
        fill_open_params(&p.open, eta);
    }
    if (!proved) return B200_OK;  // see the statuses
    rc = commit_enqueue(c, msm, srs, gs, single, 1, d_open + 1, L - 1, L, k, &pending, [&]() -> int {
        B200_CUDA(cudaMemcpyAsync(dp, hp, k * sizeof(LinkParams), cudaMemcpyHostToDevice, st));
        LinArgs a{};
        a.count = 2;
        a.p[0] = d_diff; a.pstride[0] = (uint32_t)L; a.len[0] = (uint32_t)L;
        a.p[1] = d_quot; a.pstride[1] = (uint32_t)Q; a.len[1] = (uint32_t)Q;
        a.dyn = &dp->lin_s[0];
        a.dstride = D;
        B200_LAUNCH(k_lincomb, dim3(grid_for(L, 128), k), 128, 0, st)(a, L, d_ident, L);
        HornerStrides hs;
        hs.k = k;
        hs.p = hs.s = L;
        hs.out = 1;
        hs.dyn = D;
        horner_suffix(d_ident, L, fe_zero(), d_open, d_tot, hscr, st, &dp->open, hs);
        return B200_OK;
    });
    if (rc != B200_OK) return rc;
    if ((rc = commit_collect(msm, pending, comms.data())) != B200_OK) return rc;
    for (unsigned y = 0; y < k; ++y)
        if (items[y]->status == B200_OK) items[y]->out->opening_proof = comms[y];
    if (gset && !gs) gset->proofs_seen = 1;  // both segments have run eagerly: the next call with this key captures them
    return B200_OK;
}

// Link proofs per link_chunk() call: as many as half the free device memory holds (the batch buffers the context already
// has count as free), at most kMaxBatchChunk, and below the MSM's 32-bit entry index.  Sized for the batch's longest
// polynomial and largest transform: per item the workspace, the NTT scratch and the MSM scratch of one commitment.
// B200_LINK_BATCH_CHUNK overrides it (tests: the bytes out do not depend on the chunk size).
static size_t link_batch_chunk(Context* c, const Bases* srs, const std::vector<LinkItem>& its) {
    const size_t k = its.size();
    if (const char* e = std::getenv("B200_LINK_BATCH_CHUNK")) {
        const long v = std::atol(e);
        if (v >= 1) return std::min<size_t>((size_t)v, k);
    }
    size_t L = 0, N = 0;
    for (const LinkItem& it : its) {
        L = std::max({L, it.len1, it.len2});
        N = std::max(N, (size_t)1 << it.log_N);
    }
    const MsmPlan& pl = srs->plan;
    const size_t msm_per_item = L * (size_t)pl.n_digits * 4 * 2 + ((size_t)pl.n_phys << (pl.c - 1)) * sizeof(g1_xyzz) * 4;
    const size_t per_item = (5 * L + 4 * N + 4 * (L / CH + 4 * CH + 64) + 16) * sizeof(fe) + msm_per_item;
    size_t free_b = 0, total_b = 0;
    if (cudaMemGetInfo(&free_b, &total_b) != cudaSuccess) free_b = 0;
    const Context::BatchBufs& b = c->batch;
    const size_t budget = (free_b + b.ws.cap + b.nscr.cap) / 2;
    const size_t idx_cap = ((size_t)1 << 32) / (L * (size_t)pl.n_digits) - 1;  // L * digits * chunk < 2^32
    return std::max<size_t>(1, std::min({k, kMaxBatchChunk, budget / per_item, idx_cap}));
}

// The items of a link batch on the context's batch buffers (the caller holds the context's lock): items of one transform
// size next to each other, so that a chunk divides each size's items with one launch per step.  Each item's status says
// whether its proof was made; the outputs of the others are not written.
static int link_batch_run(Context* c, const Bases* srs, std::vector<LinkItem>& its) {
    const size_t k = its.size();
    if (k == 0) return B200_OK;
    std::vector<LinkItem*> order(k);
    for (size_t i = 0; i < k; ++i) order[i] = &its[i];
    std::stable_sort(order.begin(), order.end(), [](const LinkItem* a, const LinkItem* b) { return a->log_N < b->log_N; });
    const size_t chunk = link_batch_chunk(c, srs, its);
    for (size_t off = 0; off < k; off += chunk) {
        const int rc = link_chunk(c, batch_bufs(c), srs, order.data() + off, (unsigned)std::min(chunk, k - off), /*single=*/false);
        if (rc != B200_OK) return rc;
    }
    return B200_OK;
}

}  // namespace b200

// ---------------------------------------------------------------------------------------------
// C ABI
// ---------------------------------------------------------------------------------------------
using namespace b200;

struct b200_pk {
    ProvingKey* pk;
};

namespace b200 {

// ---------------------------------------------------------------------------------------------
// settlements — the settlement arms of `NativeProofManager::handle_proof_job` (native_proof_manager.rs:514-660): prove
// the statement, then link each hint the job brings (validity first, settlement second) to the statement's hint
// ---------------------------------------------------------------------------------------------

// The link items of a settlement of the key `pk`: each caller hint first, the settlement's n + 2 coefficients second
// (a2 and comm2 are filled in once the proof is made).  Every argument check of the settlement entry points but the
// proof's own pointers: B200_ERR_INVALID, with a message that starts with `who`, before any device work.
static int settlement_items(const b200_bases* srs, const b200_pk* pk, bool witness, const b200_settlement_link* links,
                            size_t n_links, const std::string& who, std::vector<LinkItem>* its) {
    if (!srs || !pk || (n_links && !links)) {
        set_error(who + ": NULL srs, key or links");
        return B200_ERR_INVALID;
    }
    if (witness && !pk->pk->wire_vars) {
        set_error(who + ": the key holds no wiring (made by b200_plonk_preprocess, not b200_plonk_preprocess_wiring)");
        return B200_ERR_INVALID;
    }
    static const uint64_t kNoComm[8] = {};
    its->resize(n_links);
    for (size_t i = 0; i < n_links; ++i) {
        const b200_settlement_link& l = links[i];
        const std::string where = who + ": link " + std::to_string(i);
        if (!l.hint_poly || !l.hint_comm || !l.proof) {
            set_error(where + " has a NULL hint_poly, hint_comm or proof");
            return B200_ERR_INVALID;
        }
        const b200_link_item x{l.hint_poly, l.hint_len, nullptr, pk->pk->n + 2, l.hint_comm, kNoComm,
                               l.alignment, l.offset, l.size, l.proof, l.eta};
        const int rc = link_item(srs->b, x, where, &(*its)[i]);
        if (rc != B200_OK) return rc;
    }
    return B200_OK;
}

int settlement_check(const b200_bases* srs, const b200_pk* pk, bool witness, const b200_settlement_link* links, size_t n_links,
                     const char* who) {
    std::vector<LinkItem> its;
    return settlement_items(srs, pk, witness, links, n_links, who, &its);
}

// Both settlement entry points once their arguments are checked: the proof (b200_plonk_prove's path, graphs included),
// then the links as one batch against P, read where prove() left it in the single-proof workspace (proof 0's wire 0,
// n + 2 coefficients; the link batch runs in the batch buffers and does not touch it).
static int prove_settlement(b200_ctx* ctx, const Bases* srs, const ProvingKey* pk, ProveItem* item, std::vector<LinkItem>& its,
                            int* statuses, const std::string& who) {
    std::lock_guard<std::mutex> lk(ctx->c.mu);
    B200_CUDA(cudaSetDevice(ctx->c.device));
    int rc = prove(&ctx->c, single_bufs(&ctx->c), pk, item, 1, /*single=*/true);
    if (rc == B200_ERR_UNSATISFIED) {
        std::memset(item->proof, 0, sizeof(b200_proof));
        for (LinkItem& it : its) std::memset(it.out, 0, sizeof(LinkOut));
        if (statuses)
            for (size_t i = 0; i <= its.size(); ++i) statuses[i] = B200_ERR_UNSATISFIED;
        set_error(who + ": WrongQuotientPolyDegree: the settlement witness does not satisfy the circuit (no link proof made)");
        return rc;
    }
    if (rc != B200_OK) return rc;
    const fe* d_p = carve(reinterpret_cast<fe*>(ctx->c.plonk_ws.p), pk->n, 1).wpoly;
    for (LinkItem& it : its) {
        it.a2 = d_p;
        it.comm2 = item->proof->wires_poly_comms[0];
    }
    if ((rc = link_batch_run(&ctx->c, srs, its)) != B200_OK) return rc;
    if (statuses) statuses[0] = B200_OK;
    std::string bad;
    for (size_t i = 0; i < its.size(); ++i) {
        if (its[i].status != B200_OK) {
            std::memset(its[i].out, 0, sizeof(LinkOut));
            bad += (bad.empty() ? "" : ", ") + std::to_string(i);
        }
        if (statuses) statuses[1 + i] = its[i].status;
    }
    if (!bad.empty()) {
        set_error(who + ": the proof was made; the hint of link(s) " + bad +
                  " differs from the settlement's link polynomial on its group (a stale hint or a wrong layout; see statuses)");
        return B200_ERR_UNSATISFIED;
    }
    return B200_OK;
}

}  // namespace b200

extern "C" {

int b200_plonk_preprocess(b200_ctx* ctx, const b200_bases* srs, unsigned log_n, size_t num_inputs,
                          const uint64_t* selectors_evals, const uint64_t* perm, const uint64_t* k, b200_pk** out) {
    B200_TRY
    if (!ctx || !srs || !selectors_evals || !perm || !k || !out) return B200_ERR_INVALID;
    std::lock_guard<std::mutex> lk(ctx->c.mu);
    B200_CUDA(cudaSetDevice(ctx->c.device));
    ProvingKey* pk = nullptr;
    int rc = preprocess(&ctx->c, srs->b, log_n, num_inputs, reinterpret_cast<const fe*>(selectors_evals), perm, nullptr, 0,
                        reinterpret_cast<const fe*>(k), &pk);
    if (rc != B200_OK) return rc;
    *out = new b200_pk{pk};
    return B200_OK;
    B200_CATCH
}

int b200_plonk_preprocess_wiring(b200_ctx* ctx, const b200_bases* srs, unsigned log_n, size_t num_inputs,
                                 const uint64_t* selectors_evals, const unsigned* wire_vars, size_t num_vars, const uint64_t* k,
                                 b200_pk** out) {
    static_assert(sizeof(unsigned) == sizeof(uint32_t), "wire_vars holds 32-bit indices");
    B200_TRY
    if (!ctx || !srs || !selectors_evals || !wire_vars || !k || !out) return B200_ERR_INVALID;
    if (num_vars == 0 || num_vars >> 32) {
        set_error("preprocess_wiring: num_vars must be in [1, 2^32)");
        return B200_ERR_INVALID;
    }
    std::lock_guard<std::mutex> lk(ctx->c.mu);
    B200_CUDA(cudaSetDevice(ctx->c.device));
    ProvingKey* pk = nullptr;
    int rc = preprocess(&ctx->c, srs->b, log_n, num_inputs, reinterpret_cast<const fe*>(selectors_evals), nullptr,
                        reinterpret_cast<const uint32_t*>(wire_vars), num_vars, reinterpret_cast<const fe*>(k), &pk);
    if (rc != B200_OK) return rc;
    *out = new b200_pk{pk};
    return B200_OK;
    B200_CATCH
}

int b200_pk_verifying_key(const b200_pk* pk, uint64_t* selector_comms, uint64_t* sigma_comms) {
    if (!pk || !selector_comms || !sigma_comms) return B200_ERR_INVALID;
    std::memcpy(selector_comms, pk->pk->sel_comms, sizeof(pk->pk->sel_comms));
    std::memcpy(sigma_comms, pk->pk->sig_comms, sizeof(pk->pk->sig_comms));
    return B200_OK;
}

size_t b200_pk_num_inputs(const b200_pk* pk) { return pk ? pk->pk->num_inputs : 0; }
unsigned b200_pk_log_n(const b200_pk* pk) { return pk ? pk->pk->log_n : 0; }
size_t b200_pk_num_vars(const b200_pk* pk) { return pk ? pk->pk->num_vars : 0; }

int b200_plonk_link(b200_ctx* ctx, const b200_bases* srs, const uint64_t* a1, size_t len1, const uint64_t* a2,
                    size_t len2, const uint64_t* comm1, const uint64_t* comm2, unsigned alignment, size_t offset,
                    size_t size, b200_link_proof* proof, uint64_t* eta) {
    B200_TRY
    if (!ctx || !srs || !a1 || !a2 || !comm1 || !comm2 || !proof) return B200_ERR_INVALID;
    LinkItem it;
    int rc = link_item(srs->b, b200_link_item{a1, len1, a2, len2, comm1, comm2, alignment, offset, size, proof, eta}, "link", &it);
    if (rc != B200_OK) return rc;
    std::lock_guard<std::mutex> lk(ctx->c.mu);
    B200_CUDA(cudaSetDevice(ctx->c.device));
    LinkItem* one = &it;
    if ((rc = link_chunk(&ctx->c, single_bufs(&ctx->c), srs->b, &one, 1, /*single=*/true)) != B200_OK) return rc;
    if (it.status != B200_OK) {
        std::memset(proof, 0, sizeof(b200_link_proof));
        set_error("link: the two wire polynomials differ on the link group (wrong layout or mismatched witnesses)");
        return B200_ERR_UNSATISFIED;
    }
    return B200_OK;
    B200_CATCH
}

int b200_plonk_link_batch(b200_ctx* ctx, const b200_bases* srs, const b200_link_item* items, size_t k, int* statuses) {
    B200_TRY
    if (!ctx || !srs || (k && !items)) {
        set_error("plonk_link_batch: null argument");
        return B200_ERR_INVALID;
    }
    // every argument error fails the call before any device work (b200_plonk_link's B200_ERR_INVALID conditions)
    std::vector<LinkItem> its(k);
    for (size_t i = 0; i < k; ++i) {
        const b200_link_item& x = items[i];
        const std::string item = "plonk_link_batch: item " + std::to_string(i);
        if (!x.a1 || !x.a2 || !x.comm1 || !x.comm2 || !x.proof) {
            set_error(item + " has a NULL pointer");
            return B200_ERR_INVALID;
        }
        const int rc = link_item(srs->b, x, item, &its[i]);
        if (rc != B200_OK) return rc;
    }
    if (k == 0) return B200_OK;
    std::lock_guard<std::mutex> lk(ctx->c.mu);
    B200_CUDA(cudaSetDevice(ctx->c.device));
    const int rc = link_batch_run(&ctx->c, srs->b, its);
    if (rc != B200_OK) return rc;
    size_t bad = 0;
    for (size_t i = 0; i < k; ++i) {
        if (its[i].status != B200_OK) {
            std::memset(items[i].proof, 0, sizeof(b200_link_proof));
            ++bad;
        }
        if (statuses) statuses[i] = its[i].status;
    }
    if (bad) {
        set_error("plonk_link_batch: " + std::to_string(bad) + " of " + std::to_string(k) +
                  " item(s) have wire polynomials that differ on the link group (see statuses)");
        return B200_ERR_UNSATISFIED;
    }
    return B200_OK;
    B200_CATCH
}

int b200_plonk_last_timings(b200_ctx* ctx, float out_ms[8]) {
    if (!ctx || !out_ms) return B200_ERR_INVALID;
    for (int i = 0; i < 8; ++i) out_ms[i] = ctx->c.plonk_ms[i];
    return B200_OK;
}

void b200_pk_free(b200_ctx* ctx, b200_pk* pk) {
    if (!pk) return;
    if (ctx) {
        std::lock_guard<std::mutex> lk(ctx->c.mu);
        cudaSetDevice(ctx->c.device);
        cudaStreamSynchronize(ctx->c.stream);
        delete pk->pk;
    } else {
        delete pk->pk;
    }
    delete pk;
}

int b200_plonk_prove(b200_ctx* ctx, const b200_pk* pk, const uint64_t* wires, const uint64_t* pub_inputs,
                     const uint64_t* blinders, b200_proof* proof, uint64_t* link_poly, uint64_t* challenges) {
    B200_TRY
    if (!ctx || !pk || !wires || !blinders || !proof || (pk->pk->num_inputs && !pub_inputs)) return B200_ERR_INVALID;
    std::lock_guard<std::mutex> lk(ctx->c.mu);
    B200_CUDA(cudaSetDevice(ctx->c.device));
    ProveItem item{reinterpret_cast<const fe*>(wires),     reinterpret_cast<const fe*>(pub_inputs),
                   reinterpret_cast<const fe*>(blinders),  reinterpret_cast<ProofOut*>(proof),
                   reinterpret_cast<fe*>(link_poly),       reinterpret_cast<fe*>(challenges), B200_OK};
    return prove(&ctx->c, single_bufs(&ctx->c), pk->pk, &item, 1, /*single=*/true);
    B200_CATCH
}

// A key that proves from witness vectors, or B200_ERR_INVALID
static int require_wiring(const b200_pk* pk, const char* who) {
    if (pk->pk->wire_vars) return B200_OK;
    set_error(std::string(who) + ": the key holds no wiring (made by b200_plonk_preprocess, not b200_plonk_preprocess_wiring)");
    return B200_ERR_INVALID;
}

int b200_plonk_prove_witness(b200_ctx* ctx, const b200_pk* pk, const uint64_t* witness, const uint64_t* blinders,
                             b200_proof* proof, uint64_t* link_poly, uint64_t* challenges, uint64_t* pub_inputs_out) {
    B200_TRY
    if (!ctx || !pk || !witness || !blinders || !proof) return B200_ERR_INVALID;
    const int ok = require_wiring(pk, "plonk_prove_witness");
    if (ok != B200_OK) return ok;
    std::lock_guard<std::mutex> lk(ctx->c.mu);
    B200_CUDA(cudaSetDevice(ctx->c.device));
    ProveItem item{nullptr, nullptr, reinterpret_cast<const fe*>(blinders), reinterpret_cast<ProofOut*>(proof),
                   reinterpret_cast<fe*>(link_poly), reinterpret_cast<fe*>(challenges), B200_OK,
                   reinterpret_cast<const fe*>(witness), reinterpret_cast<fe*>(pub_inputs_out)};
    return prove(&ctx->c, single_bufs(&ctx->c), pk->pk, &item, 1, /*single=*/true);
    B200_CATCH
}

int b200_plonk_prove_settlement(b200_ctx* ctx, const b200_bases* srs, const b200_pk* pk, const uint64_t* wires,
                                const uint64_t* pub_inputs, const uint64_t* blinders, b200_proof* proof, uint64_t* link_poly,
                                const b200_settlement_link* links, size_t n_links, int* statuses) {
    B200_TRY
    const std::string who = "plonk_prove_settlement";
    if (!ctx || !pk || !wires || !blinders || !proof || (pk->pk->num_inputs && !pub_inputs)) {
        set_error(who + ": NULL argument");
        return B200_ERR_INVALID;
    }
    std::vector<LinkItem> its;
    const int rc = settlement_items(srs, pk, /*witness=*/false, links, n_links, who, &its);
    if (rc != B200_OK) return rc;
    ProveItem item{reinterpret_cast<const fe*>(wires),     reinterpret_cast<const fe*>(pub_inputs),
                   reinterpret_cast<const fe*>(blinders),  reinterpret_cast<ProofOut*>(proof),
                   reinterpret_cast<fe*>(link_poly),       nullptr, B200_OK};
    return prove_settlement(ctx, srs->b, pk->pk, &item, its, statuses, who);
    B200_CATCH
}

int b200_plonk_prove_settlement_witness(b200_ctx* ctx, const b200_bases* srs, const b200_pk* pk, const uint64_t* witness,
                                        const uint64_t* blinders, b200_proof* proof, uint64_t* link_poly,
                                        uint64_t* pub_inputs_out, const b200_settlement_link* links, size_t n_links,
                                        int* statuses) {
    B200_TRY
    const std::string who = "plonk_prove_settlement_witness";
    if (!ctx || !pk || !witness || !blinders || !proof) {
        set_error(who + ": NULL argument");
        return B200_ERR_INVALID;
    }
    std::vector<LinkItem> its;
    const int rc = settlement_items(srs, pk, /*witness=*/true, links, n_links, who, &its);
    if (rc != B200_OK) return rc;
    ProveItem item{nullptr, nullptr, reinterpret_cast<const fe*>(blinders), reinterpret_cast<ProofOut*>(proof),
                   reinterpret_cast<fe*>(link_poly), nullptr, B200_OK,
                   reinterpret_cast<const fe*>(witness), reinterpret_cast<fe*>(pub_inputs_out)};
    return prove_settlement(ctx, srs->b, pk->pk, &item, its, statuses, who);
    B200_CATCH
}

// The k items of a batch in chunks; statuses and return code as b200_plonk_prove_batch documents them.
static int prove_batch_items(b200_ctx* ctx, const ProvingKey* key, std::vector<ProveItem>& its, int* statuses) {
    const size_t k = its.size();
    if (k == 0) return B200_OK;
    std::lock_guard<std::mutex> lk(ctx->c.mu);
    B200_CUDA(cudaSetDevice(ctx->c.device));
    const size_t chunk = prove_batch_chunk(&ctx->c, key, k);
    for (size_t off = 0; off < k; off += chunk) {
        const unsigned cnt = (unsigned)std::min(chunk, k - off);
        const int rc = prove(&ctx->c, batch_bufs(&ctx->c), key, its.data() + off, cnt, /*single=*/false);
        if (rc != B200_OK && rc != B200_ERR_UNSATISFIED) return rc;  // B200_ERR_UNSATISFIED: every item of the chunk, see statuses
    }
    size_t bad = 0;
    for (size_t i = 0; i < k; ++i) {
        if (its[i].status != B200_OK) {
            std::memset(its[i].proof, 0, sizeof(b200_proof));
            ++bad;
        }
        if (statuses) statuses[i] = its[i].status;
    }
    if (bad) {
        set_error("WrongQuotientPolyDegree: " + std::to_string(bad) + " of " + std::to_string(k) +
                  " witnesses do not satisfy the circuit (see statuses)");
        return B200_ERR_UNSATISFIED;
    }
    return B200_OK;
}

int b200_plonk_prove_batch(b200_ctx* ctx, const b200_pk* pk, const b200_prove_item* items, size_t k, int* statuses) {
    B200_TRY
    if (!ctx || !pk || (k && !items)) return B200_ERR_INVALID;
    const ProvingKey* key = pk->pk;
    std::vector<ProveItem> its(k);
    for (size_t i = 0; i < k; ++i) {
        const b200_prove_item& x = items[i];
        if (!x.wires || !x.blinders || !x.proof || (key->num_inputs && !x.pub_inputs)) {
            set_error("plonk_prove_batch: item " + std::to_string(i) + " has a NULL pointer");
            return B200_ERR_INVALID;
        }
        its[i] = ProveItem{reinterpret_cast<const fe*>(x.wires), reinterpret_cast<const fe*>(x.pub_inputs),
                           reinterpret_cast<const fe*>(x.blinders), reinterpret_cast<ProofOut*>(x.proof),
                           reinterpret_cast<fe*>(x.link_poly), reinterpret_cast<fe*>(x.challenges), B200_OK};
    }
    return prove_batch_items(ctx, key, its, statuses);
    B200_CATCH
}

int b200_plonk_prove_witness_batch(b200_ctx* ctx, const b200_pk* pk, const b200_witness_item* items, size_t k, int* statuses) {
    B200_TRY
    if (!ctx || !pk || (k && !items)) return B200_ERR_INVALID;
    const int ok = require_wiring(pk, "plonk_prove_witness_batch");
    if (ok != B200_OK) return ok;
    std::vector<ProveItem> its(k);
    for (size_t i = 0; i < k; ++i) {
        const b200_witness_item& x = items[i];
        if (!x.witness || !x.blinders || !x.proof) {
            set_error("plonk_prove_witness_batch: item " + std::to_string(i) + " has a NULL pointer");
            return B200_ERR_INVALID;
        }
        its[i] = ProveItem{nullptr, nullptr, reinterpret_cast<const fe*>(x.blinders), reinterpret_cast<ProofOut*>(x.proof),
                           reinterpret_cast<fe*>(x.link_poly), reinterpret_cast<fe*>(x.challenges), B200_OK,
                           reinterpret_cast<const fe*>(x.witness), reinterpret_cast<fe*>(x.pub_inputs_out)};
    }
    return prove_batch_items(ctx, pk->pk, its, statuses);
    B200_CATCH
}


/* ---- device-vector primitives (collaborative prover) ---------------------------------------------------------- */
int b200_fr_vec_op(b200_ctx* ctx, int op, const void* d_a, const void* d_b, int b_is_scalar, size_t n, void* d_out) {
    B200_TRY
    if (!ctx || op < 0 || op > 2 || (n && (!d_a || !d_b || !d_out))) return B200_ERR_INVALID;
    if (n == 0) return B200_OK;
    std::lock_guard<std::mutex> lk(ctx->c.mu);
    B200_CUDA(cudaSetDevice(ctx->c.device));
    B200_LAUNCH(k_fr_vec_op, grid_for(n, 256), 256, 0, ctx->c.stream)(op, reinterpret_cast<const fe*>(d_a), reinterpret_cast<const fe*>(d_b),
                                                                     b_is_scalar, n, reinterpret_cast<fe*>(d_out));
    B200_CUDA(cudaGetLastError());
    B200_CUDA(cudaStreamSynchronize(ctx->c.stream));
    return B200_OK;
    B200_CATCH
}

int b200_fr_batch_inverse_device(b200_ctx* ctx, void* d_data, size_t n) {
    B200_TRY
    if (!ctx || (n && !d_data)) return B200_ERR_INVALID;
    if (n == 0) return B200_OK;
    std::lock_guard<std::mutex> lk(ctx->c.mu);
    B200_CUDA(cudaSetDevice(ctx->c.device));
    int rc = ctx->c.ntt_scratch.reserve(n * sizeof(fe));
    if (rc != B200_OK) return rc;
    batch_inverse_enqueue(nullptr, reinterpret_cast<fe*>(d_data), reinterpret_cast<fe*>(ctx->c.ntt_scratch.p), n, ctx->c.stream);
    B200_CUDA(cudaGetLastError());
    B200_CUDA(cudaStreamSynchronize(ctx->c.stream));
    return B200_OK;
    B200_CATCH
}

int b200_fr_poly_eval_device(b200_ctx* ctx, const void* d_coeffs, size_t len, const uint64_t z[4], uint64_t out[4]) {
    B200_TRY
    if (!ctx || !z || !out || (len && !d_coeffs)) return B200_ERR_INVALID;
    if (len == 0) {
        std::memset(out, 0, 32);
        return B200_OK;
    }
    std::lock_guard<std::mutex> lk(ctx->c.mu);
    B200_CUDA(cudaSetDevice(ctx->c.device));
    int rc = ctx->c.plonk_ws.reserve((2 * (len / CH + len / CH / CH) + 4 * CH + 64) * sizeof(fe));
    if (rc != B200_OK) return rc;
    fe* scr = reinterpret_cast<fe*>(ctx->c.plonk_ws.p);
    fe zz;
    std::memcpy(&zz, z, 32);
    const fe* polys[1] = {reinterpret_cast<const fe*>(d_coeffs)};
    const size_t lens[1] = {len};
    eval_batch(polys, lens, &zz, 1, scr, scr + 8, ctx->c.stream);
    B200_CUDA(cudaMemcpyAsync(out, scr, 32, cudaMemcpyDeviceToHost, ctx->c.stream));
    B200_CUDA(cudaStreamSynchronize(ctx->c.stream));
    return B200_OK;
    B200_CATCH
}

int b200_fr_poly_div_linear_device(b200_ctx* ctx, const void* d_p, size_t len, const uint64_t z[4], void* d_q) {
    B200_TRY
    if (!ctx || !z || len < 2 || !d_p || !d_q) return B200_ERR_INVALID;
    std::lock_guard<std::mutex> lk(ctx->c.mu);
    B200_CUDA(cudaSetDevice(ctx->c.device));
    const size_t L = len + 8;
    int rc = ctx->c.plonk_ws.reserve((L + 4 * (L / CH + 4 * CH + 64) + 16) * sizeof(fe));
    if (rc != B200_OK) return rc;
    fe* S = reinterpret_cast<fe*>(ctx->c.plonk_ws.p);
    fe* hscr = S + L;
    fe* slot = hscr + 4 * (L / CH + 4 * CH + 64);
    fe zz;
    std::memcpy(&zz, z, 32);
    horner_suffix(reinterpret_cast<const fe*>(d_p), len, zz, S, slot, hscr, ctx->c.stream);
    B200_CUDA(cudaMemcpyAsync(d_q, S + 1, (len - 1) * sizeof(fe), cudaMemcpyDeviceToDevice, ctx->c.stream));  // drop the remainder S[0]
    B200_CUDA(cudaStreamSynchronize(ctx->c.stream));
    return B200_OK;
    B200_CATCH
}

}  // extern "C"
