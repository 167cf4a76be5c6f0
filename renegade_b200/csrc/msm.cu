// Pippenger multi-scalar multiplication on BN254 G1 for sm_90a.
//
// Replaces what the reference reaches through jf-primitives `UnivariateKzgPCS::commit` ->
// ark-ec 0.4.2 `VariableBaseMSM::msm_bigint(&powers_of_g, &coeffs)` (call sites
// /root/reference/crates/circuits/circuit-types/src/traits.rs:850,996 and
// circuits-core/src/zk_circuits/proof_linking/intent_only.rs:42-47; algorithm restated in
// SURVEY.md App. B).  The result is a group element, so after affine normalisation it is
// bit-identical to arkworks' whatever the bucket schedule.
//
// Device-first design (not arkworks' per-window rayon loop):
//   * bases are fixed (the SRS), HBM is large (80 GB on an H100): at load time every base gets its window
//     multiples 2^(c*j)*P precomputed, so ALL windows share ONE bucket set — no per-window
//     reduction, no Horner doublings on the device; the tables are gathered at 64 B/point
//     (two full sectors), well inside the HBM budget of an integer-pipe-bound kernel;
//   * signed c-bit digits halve the bucket count;
//   * digits are counting-sorted by bucket (histogram -> scan -> scatter, L2-resident atomics),
//     then one thread per bucket folds its points with XYZZ mixed additions (8M+2S, no
//     inversion), prefetching the next 64-byte point while the current addition runs;
//   * sum_k (k+1) B_k without a running sum: the buckets of a window form a matrix whose row and
//     column sums carry the weights, so every bucket enters two plain additions (one serial level of
//     fan-in 8 / 4, then the rest of each row / column), and the two weighted sums that remain become
//     c - 1 per-bit sums.  Throughput plans (the prover's batched commitments) read the buckets from
//     their segment sums in the serial level and finish with two wide levels of warp-local sums;
//     latency plans (one MSM alone) combine the buckets first and finish with shared-memory binary
//     trees whose dependent additions run on four lanes each (xyzz_add_quad).  The last ~2 KB go to
//     the host, which runs the Horner over the bit sums and the single field inversion of the batch.
#include <algorithm>
#include <cstdlib>
#include <vector>

#include "device_ctx.h"
#include "ec.cuh"

namespace b200 {

namespace {

constexpr uint32_t kIdxBits = 26;  // entry = sign(1) | table(5) | point index(26)
constexpr uint32_t kIdxMask = (1u << kIdxBits) - 1u;
#ifndef B200_SEG_LEN
#define B200_SEG_LEN 32
#endif
constexpr int kSegLen = B200_SEG_LEN;  // a bucket is folded in segments of at most this many points
constexpr int kCombineSeq = 64;    // buckets with more segments than this take the block-tree path
constexpr int kReduceThreads = 128;  // block size of the heavy-bucket tree

// ---- scalar digits ---------------------------------------------------------------------------
__device__ __forceinline__ uint32_t get_bits(const uint32_t* s, int pos, int c) {
    const int limb = pos >> 5, off = pos & 31;
    uint32_t v = limb < 8 ? s[limb] >> off : 0u;
    if (off + c > 32 && limb + 1 < 8) v |= s[limb + 1] << (32 - off);
    return v & ((1u << c) - 1u);
}

// Calls f(bucket, code) for every non-zero signed digit of scalar i.
template <class F>
__device__ __forceinline__ void for_each_digit(const fe* scalars, size_t i, int montgomery,
                                               const MsmPlan& pl, uint32_t point_idx, F f) {
    fe s = fe_load_ro(scalars + i);
    if (montgomery) s = fe_from_mont<FrCfg>(s);
    uint32_t limbs[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) limbs[k] = s.l[k];
    const uint32_t half = 1u << (pl.c - 1);
    uint32_t carry = 0;
    for (int w = 0; w < pl.n_digits; ++w) {
        uint32_t raw = get_bits(limbs, w * pl.c, pl.c) + carry;
        uint32_t neg = 0, mag = raw;
        if (raw > half) {  // digit = raw - 2^c  (magnitude 2^c - raw, possibly 0 when raw = 2^c)
            mag = (1u << pl.c) - raw;
            neg = 1;
            carry = 1;
        } else {
            carry = 0;
        }
        if (mag == 0) continue;
        const uint32_t phys = (uint32_t)(w % pl.n_phys), table = (uint32_t)(w / pl.n_phys);
        const uint32_t bucket = phys * half + (mag - 1u);
        f(bucket, (neg << 31) | (table << kIdxBits) | point_idx);
    }
}

// blockIdx.y = index of the MSM inside a batch (same bases, `stride` scalars apart); every MSM owns
// its own range of `buckets_per_msm` buckets, so the later phases see one big bucket array.
__global__ void msm_count_kernel(const fe* scalars, size_t n, size_t stride, int montgomery, MsmPlan pl,
                                 uint32_t buckets_per_msm, uint32_t* counts) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint32_t* my = counts + (size_t)blockIdx.y * buckets_per_msm;
    for_each_digit(scalars + (size_t)blockIdx.y * stride, i, montgomery, pl, (uint32_t)i,
                   [&](uint32_t bucket, uint32_t) { atomicAdd(my + bucket, 1u); });
}

__global__ void msm_scatter_kernel(const fe* scalars, size_t n, size_t stride, int montgomery, MsmPlan pl,
                                   uint32_t base_off, uint32_t buckets_per_msm, uint32_t* cursor,
                                   uint32_t* entries) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint32_t* my = cursor + (size_t)blockIdx.y * buckets_per_msm;
    for_each_digit(scalars + (size_t)blockIdx.y * stride, i, montgomery, pl, (uint32_t)i + base_off,
                   [&](uint32_t bucket, uint32_t code) {
                       const uint32_t pos = atomicAdd(my + bucket, 1u);
                       entries[pos] = code;
                   });
}

// ---- fused single-pass scan of the bucket histogram ------------------------------------------------
// One launch produces everything the later phases need from the histogram: the exclusive scan of the
// counts (`offsets`, and its copy `cursor` for the scatter), the exclusive scan of the per-bucket segment
// counts ceil(count / kSegLen) (`seg_offsets`), the histogram of segment lengths turned into start
// offsets, longest first (`seg_starts`, the cursor of msm_segorder_kernel), and the clean-up for the next
// MSM on this scratch (counts, heavy-bucket counter, tile statuses and tickets back to zero).
// Single-pass chained scan with decoupled look-back: tiles are handed out by an atomic ticket (so a tile's
// predecessors are always running or done), every tile publishes its aggregate and then its inclusive
// prefix in one 64-bit status word (flag:2 | segments:30 | entries:32), and warp 0 of a tile looks back
// over 32 predecessors at a time.  The block that finishes last owns the epilogue.
constexpr int kScanThreads = 256;
constexpr int kScanItems = 16;
constexpr int kScanTile = kScanThreads * kScanItems;
constexpr uint32_t kSegBins = kSegLen + 1;

struct ScanState {          // zero-initialised when the scratch is allocated; left zeroed by every launch
    uint32_t ticket, done;
    uint32_t seg_hist[kSegBins + 1];
    uint32_t seg_starts[kSegBins + 1];
    uint32_t heavy_count;
    uint32_t pad[3];
    // followed by n_tiles 64-bit status words (8-byte aligned: the header is 4 * (2 + 34 + 34 + 4) = 296 bytes)
};
static_assert(sizeof(ScanState) % 8 == 0, "status words are 8-byte aligned");

__device__ __forceinline__ uint64_t status_pack(uint32_t flag, uint32_t a, uint32_t b) {
    return ((uint64_t)flag << 62) | ((uint64_t)b << 32) | a;
}
__device__ __forceinline__ uint64_t ld_status(const uint64_t* p) {
    uint64_t v;
    asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_status(uint64_t* p, uint64_t v) {
    asm volatile("st.relaxed.gpu.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}

__global__ void __launch_bounds__(kScanThreads) msm_scan_kernel(uint32_t* __restrict__ counts, uint32_t n, uint32_t n_tiles,
                                                                ScanState* __restrict__ stt, uint64_t* __restrict__ status,
                                                                uint32_t* __restrict__ offsets, uint32_t* __restrict__ cursor,
                                                                uint32_t* __restrict__ seg_offsets) {
    __shared__ uint32_t s_tile, s_last;
    __shared__ uint32_t s_hist[kSegBins];
    __shared__ uint32_t s_wa[kScanThreads / 32], s_wb[kScanThreads / 32];
    __shared__ uint32_t s_pa, s_pb;  // exclusive prefix of this tile
    const uint32_t tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    if (tid == 0) s_tile = atomicAdd(&stt->ticket, 1u);
    if (tid < kSegBins) s_hist[tid] = 0;
    __syncthreads();
    const uint32_t tile = s_tile;
    const uint32_t base = tile * kScanTile + tid * kScanItems;
    // n is a multiple of 16 (buckets per window are a power of two >= 32): a thread's items are all in or all out
    uint32_t v[kScanItems], sv[kScanItems];
    uint32_t a = 0, b = 0;
    const bool in = base < n;
    if (in) {
        uint4* src = reinterpret_cast<uint4*>(counts + base);
#pragma unroll
        for (int k = 0; k < kScanItems / 4; ++k) {
            const uint4 q = src[k];
            v[4 * k] = q.x; v[4 * k + 1] = q.y; v[4 * k + 2] = q.z; v[4 * k + 3] = q.w;
            src[k] = make_uint4(0u, 0u, 0u, 0u);  // the histogram is consumed: leave it zeroed for the next MSM
        }
#pragma unroll
        for (int k = 0; k < kScanItems; ++k) {
            const uint32_t cnt = v[k];
            const uint32_t segs = (cnt + (uint32_t)kSegLen - 1u) / (uint32_t)kSegLen;
            sv[k] = segs;
            a += cnt;
            b += segs;
            if (segs) {  // near-equal split: rem segments of len + 1, the others of len
                const uint32_t len = cnt / segs, rem = cnt % segs;
                atomicAdd(&s_hist[len], segs - rem);
                if (rem) atomicAdd(&s_hist[len + 1], rem);
            }
        }
    } else {
#pragma unroll
        for (int k = 0; k < kScanItems; ++k) v[k] = sv[k] = 0;
    }
    // block-wide exclusive scan of the (a, b) pairs
    uint32_t ia = a, ib = b;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const uint32_t ta = __shfl_up_sync(0xffffffffu, ia, d), tb = __shfl_up_sync(0xffffffffu, ib, d);
        if ((int)lane >= d) { ia += ta; ib += tb; }
    }
    if (lane == 31) { s_wa[wid] = ia; s_wb[wid] = ib; }
    __syncthreads();
    if (wid == 0) {
        const uint32_t wa = lane < kScanThreads / 32 ? s_wa[lane] : 0u, wb = lane < kScanThreads / 32 ? s_wb[lane] : 0u;
        uint32_t xa = wa, xb = wb;
#pragma unroll
        for (int d = 1; d < kScanThreads / 32; d <<= 1) {
            const uint32_t ta = __shfl_up_sync(0xffffffffu, xa, d), tb = __shfl_up_sync(0xffffffffu, xb, d);
            if ((int)lane >= d) { xa += ta; xb += tb; }
        }
        if (lane < kScanThreads / 32) { s_wa[lane] = xa - wa; s_wb[lane] = xb - wb; }
        const uint32_t tot_a = __shfl_sync(0xffffffffu, xa, kScanThreads / 32 - 1);
        const uint32_t tot_b = __shfl_sync(0xffffffffu, xb, kScanThreads / 32 - 1);
        // decoupled look-back
        uint32_t pa = 0, pb = 0;
        if (tile == 0) {
            if (lane == 0) st_status(status, status_pack(2u, tot_a, tot_b));
        } else {
            if (lane == 0) st_status(status + tile, status_pack(1u, tot_a, tot_b));
            int look = (int)tile - 1;  // lane l inspects tile look - l
            while (true) {
                const int t = look - (int)lane;
                uint64_t w = 0;
                if (t >= 0) {
                    do { w = ld_status(status + t); } while ((w >> 62) == 0);
                } else {
                    w = status_pack(2u, 0u, 0u);  // before tile 0: an empty inclusive prefix
                }
                const uint32_t is_prefix = __ballot_sync(0xffffffffu, (w >> 62) == 2u);
                const int stop = __ffs(is_prefix) - 1;  // nearest tile that already knows its inclusive prefix
                // no prefix among the 32 inspected tiles (stop < 0): all of their aggregates count and the window moves on
                const bool take = stop < 0 || (int)lane <= stop;
                uint32_t ca = take ? (uint32_t)w : 0u, cb = take ? (uint32_t)(w >> 32) & 0x3fffffffu : 0u;
#pragma unroll
                for (int d = 16; d > 0; d >>= 1) {
                    ca += __shfl_xor_sync(0xffffffffu, ca, d);
                    cb += __shfl_xor_sync(0xffffffffu, cb, d);
                }
                pa += ca;
                pb += cb;
                if (stop >= 0) break;  // (always true once the window reaches below tile 0)
                look -= 32;
            }
            if (lane == 0) st_status(status + tile, status_pack(2u, pa + tot_a, pb + tot_b));
        }
        if (lane == 0) { s_pa = pa; s_pb = pb; }
    }
    __syncthreads();
    if (in) {
        uint32_t ea = s_pa + s_wa[wid] + (ia - a), eb = s_pb + s_wb[wid] + (ib - b);
#pragma unroll
        for (int k = 0; k < kScanItems; ++k) {
            offsets[base + k] = ea;
            cursor[base + k] = ea;
            seg_offsets[base + k] = eb;
            ea += v[k];
            eb += sv[k];
        }
        if (base + kScanItems == n) {  // the last in-range thread closes both arrays
            offsets[n] = ea;
            seg_offsets[n] = eb;
        }
    }
    if (tid < kSegBins && s_hist[tid]) atomicAdd(&stt->seg_hist[tid], s_hist[tid]);
    __threadfence();
    __syncthreads();
    if (tid == 0) s_last = atomicAdd(&stt->done, 1u) == n_tiles - 1 ? 1u : 0u;
    __syncthreads();
    if (s_last) {  // every tile has finished its look-back and added its segment histogram
        __threadfence();
        for (uint32_t t = tid; t < n_tiles; t += kScanThreads) status[t] = 0;
        if (tid == 0) {
            uint32_t run = 0;
            for (int l = kSegLen; l >= 0; --l) {  // start offsets, longest segments first
                const uint32_t c = reinterpret_cast<volatile uint32_t*>(stt->seg_hist)[l];
                stt->seg_starts[l] = run;
                run += c;
            }
            for (uint32_t l = 0; l < kSegBins; ++l) stt->seg_hist[l] = 0;
            stt->heavy_count = 0;
            stt->ticket = 0;
            stt->done = 0;
        }
    }
}

// ---- bucket accumulation ---------------------------------------------------------------------------
// Buckets are folded in SEGMENTS of at most kSegLen sorted entries (a bucket of k entries is cut
// into ceil(k / kSegLen) near-equal segments), one thread per segment, so the work per thread is
// bounded whatever the digit distribution: the top window of a 254-bit scalar, small witness
// values or repeated scalars all pile points into a few buckets.
__device__ __forceinline__ g1_affine load_entry_point(const g1_affine* tables, size_t n,
                                                      uint32_t code) {
    const size_t idx = code & kIdxMask, table = (code >> kIdxBits) & 31u;
    return g1_affine_load_ro(tables + table * n + idx);
}

// Segment lengths differ (Poisson bucket sizes); lanes of a warp that fold different numbers of
// points idle in lockstep.  A counting sort of the segment ids by length (kSegLen + 1 bins, longest
// first; bin starts from msm_scan_kernel) hands every warp segments of equal length.  One thread per
// bucket: a bucket of cnt entries in k segments has rem = cnt % k segments of cnt / k + 1 entries, then
// k - rem of cnt / k.  Slots are claimed per block (shared-memory ranks, one global atomic per block and
// length) and the same thread records seg_bucket[s] = bucket owning segment s.  Buckets cut into more than kCombineSeq
// segments are listed for msm_heavy_combine_kernel.
__global__ void __launch_bounds__(256) msm_segorder_kernel(const uint32_t* __restrict__ offsets,
                                                           const uint32_t* __restrict__ seg_offsets, uint32_t n_buckets,
                                                           uint32_t* __restrict__ seg_cursor /* kSegBins */,
                                                           uint32_t* __restrict__ seg_bucket, uint32_t* __restrict__ order,
                                                           uint32_t* __restrict__ heavy_count, uint32_t* __restrict__ heavy_list) {
    __shared__ uint32_t s_cnt[kSegBins], s_base[kSegBins];
    if (threadIdx.x < kSegBins) s_cnt[threadIdx.x] = 0;
    __syncthreads();
    const uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t k = 0, s0 = 0, len = 0, rem = 0, r0 = 0, r1 = 0;
    if (b < n_buckets) {
        s0 = seg_offsets[b];
        k = seg_offsets[b + 1] - s0;
        if (k) {
            const uint32_t cnt = offsets[b + 1] - offsets[b];
            len = cnt / k;
            rem = cnt % k;
            r0 = atomicAdd(&s_cnt[len], k - rem);
            if (rem) r1 = atomicAdd(&s_cnt[len + 1], rem);
        }
        if (k > (uint32_t)kCombineSeq) heavy_list[atomicAdd(heavy_count, 1u)] = b;
    }
    __syncthreads();
    if (threadIdx.x < kSegBins && s_cnt[threadIdx.x]) s_base[threadIdx.x] = atomicAdd(&seg_cursor[threadIdx.x], s_cnt[threadIdx.x]);
    __syncthreads();
    if (k) {
        const uint32_t slot1 = rem ? s_base[len + 1] + r1 : 0u, slot0 = s_base[len] + r0;
        for (uint32_t j = 0; j < k; ++j) {
            seg_bucket[s0 + j] = b;
            order[j < rem ? slot1 + j : slot0 + (j - rem)] = s0 + j;
        }
    }
}

__global__ void __launch_bounds__(128) msm_accumulate_kernel(const uint32_t* __restrict__ entries,
                                                             const uint32_t* __restrict__ offsets,
                                                             const uint32_t* __restrict__ seg_offsets,
                                                             const uint32_t* __restrict__ seg_bucket,
                                                             const uint32_t* __restrict__ order,
                                                             const g1_affine* __restrict__ tables,
                                                             size_t n_points, uint32_t n_buckets,
                                                             g1_xyzz* __restrict__ seg_sums) {
    const uint32_t tid = blockIdx.x * blockDim.x + threadIdx.x;
    if (tid >= seg_offsets[n_buckets]) return;  // the grid is sized for the worst case
    const uint32_t s = order[tid];
    const uint32_t b = seg_bucket[s];
    const uint32_t j = s - seg_offsets[b], k = seg_offsets[b + 1] - seg_offsets[b];
    const uint32_t first = offsets[b], cnt = offsets[b + 1] - first;
    const uint32_t base = cnt / k, rem = cnt % k;  // near-equal split of the bucket
    uint32_t e = first + j * base + min(j, rem);
    const uint32_t end = e + base + (j < rem ? 1u : 0u);
    g1_xyzz acc = g1_xyzz_inf();
    if (e < end) {
        uint32_t code = entries[e];
        g1_affine next = load_entry_point(tables, n_points, code);
        while (true) {
            g1_affine cur = next;
            const uint32_t cur_code = code;
            ++e;
            if (e < end) {  // prefetch the next point under the current addition
                code = entries[e];
                next = load_entry_point(tables, n_points, code);
            }
            if (cur_code >> 31) cur.y = fe_neg<FqCfg>(cur.y);
            acc = g1_add_mixed(acc, cur);
            if (e >= end) break;
        }
    }
    g1_xyzz_store(seg_sums + s, acc);
}

// The reduction-side kernels run one warp per SM sub-partition on long dependent chains; with
// g1_add inlined a dozen times their code no longer fits the instruction cache (the profiler shows
// "no instruction" stalls).  Out-of-line copies keep those kernels small.
__device__ __noinline__ g1_xyzz xyzz_add(const g1_xyzz& a, const g1_xyzz& b) { return g1_add(a, b); }

// ---- one XYZZ addition by the four lanes of a quad ------------------------------------------------------------
// The tails of the bucket reduction are chains of DEPENDENT additions with almost nobody else on the SM: one lane
// walks through the 14 field products of g1_add one after the other while the lanes beside it idle.  The 14 products are only
// four deep, so a quad (lanes 4k .. 4k+3) takes one product per lane and stage and trades the results by shuffle:
//   stage 1   u1 = X1*ZZ2      u2 = X2*ZZ1     s1 = Y1*ZZZ2      s2 = Y2*ZZZ1        P = u2 - u1, R = s2 - s1
//   stage 2   pp = P^2         r2 = R^2        zz = ZZ1*ZZ2      zzz = ZZZ1*ZZZ2
//   stage 3   ppp = P*pp       q = u1*pp       ZZ3 = zz*pp       w = zzz*pp          X3 = r2 - ppp - 2q
//   stage 4   t1 = R*(q - X3)  t2 = s1*ppp     (nothing)         ZZZ3 = w*P          Y3 = t1 - t2
// (same formulas as g1_add, EFD add-2008-s, with Y3 as two products instead of the fused pair — any correct group
// addition gives the same affine point).  Operands live in shared memory as arrays of four field elements; the sum
// replaces operand a.  Identity operands and P = 0 (doubling / cancellation) are decided identically by the four lanes
// and take the exact paths of g1_add.  All 32 lanes of a warp call this together (the shuffles are warp-wide): quads
// with nothing to add pass on = false and operands nobody writes during the call.
__device__ __forceinline__ fe fe_quad_bcast(const fe& v, int src) {
    fe r;
#pragma unroll
    for (int k = 0; k < 8; ++k) r.l[k] = __shfl_sync(0xffffffffu, v.l[k], src, 4);
    return r;
}
__device__ __forceinline__ fe fe_pick3(uint32_t q, const fe& a0, const fe& a1, const fe& rest) {  // q = 0 ? a0 : q = 1 ? a1 : rest
    fe r;
#pragma unroll
    for (int k = 0; k < 8; ++k) r.l[k] = q == 0u ? a0.l[k] : (q == 1u ? a1.l[k] : rest.l[k]);
    return r;
}
__device__ __forceinline__ void xyzz_add_quad(g1_xyzz* sh, uint32_t ia, uint32_t ib, bool on) {
    fe* F = reinterpret_cast<fe*>(sh);  // point i = F[4 i .. 4 i + 3] = x, y, zz, zzz
    const uint32_t q = threadIdx.x & 3u;
    const uint32_t hi = q | 2u;  // lanes 2 and 3 multiply the zz / zzz pair in stage 2
    const fe a_hi = fe_load(F + 4u * ia + hi), b_hi = fe_load(F + 4u * ib + hi);
    const bool a_inf = fe_is_zero(fe_load(F + 4u * ia + 2u)), b_inf = fe_is_zero(fe_load(F + 4u * ib + 2u));
    // nothing but copies in the whole warp (empty slots of a padded tree): skip the arithmetic
    if (__all_sync(0xffffffffu, !on || a_inf || b_inf)) {
        __syncwarp();  // the quad's reads of a above, before its lanes overwrite a
        if (on && a_inf && !b_inf) fe_store(F + 4u * ia + q, fe_load(F + 4u * ib + q));
        return;
    }
    // stage 1: lane 0 X1*ZZ2, lane 1 X2*ZZ1, lane 2 Y1*ZZZ2, lane 3 Y2*ZZZ1
    const uint32_t i1 = (q & 1u) ? ib : ia, i2 = (q & 1u) ? ia : ib;
    const fe m1 = fe_mul<Fq>(fe_load(F + 4u * i1 + (q >> 1)), fe_load(F + 4u * i2 + 2u + (q >> 1)));
    const fe u1 = fe_quad_bcast(m1, 0), u2 = fe_quad_bcast(m1, 1), s1 = fe_quad_bcast(m1, 2), s2 = fe_quad_bcast(m1, 3);
    const fe pd = fe_sub<Fq>(u2, u1), rd = fe_sub<Fq>(s2, s1);
    const bool p0 = fe_is_zero(pd);
    // stage 2
    const fe m2 = fe_mul<Fq>(fe_pick3(q, pd, rd, a_hi), fe_pick3(q, pd, rd, b_hi));
    const fe pp = fe_quad_bcast(m2, 0);
    // stage 3
    const fe m3 = fe_mul<Fq>(fe_pick3(q, pd, u1, m2), pp);
    const fe ppp = fe_quad_bcast(m3, 0), qq = fe_quad_bcast(m3, 1), r2 = fe_quad_bcast(m2, 1);
    const fe x3 = fe_sub<Fq>(fe_sub<Fq>(r2, ppp), fe_dbl<Fq>(qq));
    // stage 4 (lane 2's product is not used)
    const fe m4 = fe_mul<Fq>(fe_pick3(q, rd, s1, m3), fe_pick3(q, fe_sub<Fq>(qq, x3), ppp, pd));
    const fe t2 = fe_quad_bcast(m4, 1);
    // every lane of the warp has passed its last read of the operands; the barrier orders those reads before the
    // stores that replace a (a shuffle synchronises execution, not shared memory)
    __syncwarp();
    if (!on || b_inf) return;
    if (a_inf) {
        fe_store(F + 4u * ia + q, fe_load(F + 4u * ib + q));
    } else if (p0) {  // a = +-b: exact doubling / identity, by one lane
        if (q == 0u) {
            const g1_xyzz r = xyzz_add(sh[ia], sh[ib]);
            sh[ia] = r;
        }
    } else if (q == 0u) {
        fe_store(F + 4u * ia, x3);
        fe_store(F + 4u * ia + 1u, fe_sub<Fq>(m4, t2));
    } else if (q == 2u) {
        fe_store(F + 4u * ia + 2u, m3);
    } else if (q == 3u) {
        fe_store(F + 4u * ia + 3u, m4);
    }
}

// bucket = sum of its segment sums: sequential for ordinary buckets, left to a block tree
// (msm_heavy_combine_kernel) for buckets cut into more than kCombineSeq segments.  Latency plans only: a throughput
// plan's serial tree level reads the segment sums itself (bucket_first).
__global__ void __launch_bounds__(128) msm_bucket_combine_kernel(const g1_xyzz* __restrict__ seg_sums,
                                                                 const uint32_t* __restrict__ seg_offsets,
                                                                 uint32_t n_buckets,
                                                                 g1_xyzz* __restrict__ buckets) {
    const uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= n_buckets) return;
    const uint32_t s0 = seg_offsets[b], s1 = seg_offsets[b + 1];
    if (s1 - s0 > (uint32_t)kCombineSeq) return;
    g1_xyzz acc = g1_xyzz_inf();
    if (s0 < s1) {
        acc = g1_xyzz_load(seg_sums + s0);
        for (uint32_t s = s0 + 1; s < s1; ++s) acc = xyzz_add(acc, g1_xyzz_load(seg_sums + s));
    }
    g1_xyzz_store(buckets + b, acc);
}

__global__ void __launch_bounds__(kReduceThreads) msm_heavy_combine_kernel(const g1_xyzz* __restrict__ seg_sums,
                                                                           const uint32_t* __restrict__ seg_offsets,
                                                                           const uint32_t* __restrict__ heavy_count,
                                                                           const uint32_t* __restrict__ heavy_list,
                                                                           g1_xyzz* __restrict__ buckets) {
    __shared__ g1_xyzz sh[kReduceThreads];
    for (uint32_t h = blockIdx.x; h < *heavy_count; h += gridDim.x) {
        const uint32_t b = heavy_list[h];
        const uint32_t s0 = seg_offsets[b], s1 = seg_offsets[b + 1];
        g1_xyzz acc = g1_xyzz_inf();
        for (uint32_t s = s0 + threadIdx.x; s < s1; s += blockDim.x) acc = xyzz_add(acc, g1_xyzz_load(seg_sums + s));
        sh[threadIdx.x] = acc;
        __syncthreads();
        for (int stride = kReduceThreads / 2; stride > 0; stride >>= 1) {
            if ((int)threadIdx.x < stride) sh[threadIdx.x] = xyzz_add(sh[threadIdx.x], sh[threadIdx.x + stride]);
            __syncthreads();
        }
        if (threadIdx.x == 0) g1_xyzz_store(buckets + b, sh[0]);
        __syncthreads();
    }
}

// ---- bucket reduction: sum_k (k+1) * B[k] per physical window -----------------------------------
// View a window's H = 2^(c-1) buckets as a matrix M[hi][lo] with L = 2^l columns (k = hi * L + lo):
//     sum_k (k + 1) B[k] = L * sum_hi hi * R[hi] + sum_lo (lo + 1) * C[lo],
// R = row sums, C = column sums.  Every bucket enters exactly two additions (its row tree and its column
// tree), and the trees are plain sums: all of their work is data-parallel with dependent chains of at most
// 7 additions per level (fan-in <= 8) — instead of a running sum whose chain is as long as a thread's chunk.
// What is left is two weighted sums over 2^l / 2^(c-1-l) elements (<= 256 each up to c = 17), written as c - 1 bit
// sums: msm_tail_bits_kernel (throughput plans) or msm_bitsum_kernel (latency plans), then msm_horner_kernel or the host.
//   msm_tree_kernel, one launch per level, both trees side by side:
//     out[a * inner + b] = sum_{j < T} in[(a * T + j) * inner + b]
//   row tree: inner = 1 (sums of T neighbours over the flat bucket array; L is a multiple of every T, so a
//   group never straddles a row or a window); column tree: inner = L (sums of T consecutive rows).
struct TreeLevel {
    const g1_xyzz* in;
    g1_xyzz* out;
    uint32_t n_out, t_log, inner_log, n_blocks;
};
struct TreeArgs {
    TreeLevel row, col;
    // throughput plans: the serial level reads the buckets from the accumulation's segment sums (the bucket combine folded
    // in); nullptr: from the combined buckets in `in` (latency plans, msm_bucket_combine_kernel)
    const uint32_t* seg_offsets;
    const g1_xyzz* seg_sums;
};
constexpr int kTreeThreads = 128;
constexpr size_t kSmallTreeBuckets = (size_t)1 << 17;  // latency plans up to this many buckets: fan-in 4 in the serial level, see tree_shape
constexpr size_t kQuadTreeMaxOutputs = 16384;  // msm_tree_quad_kernel up to this many outputs (65536 lanes), see msm_launch_batch

// Bucket bk's first segment sum (the identity for an empty bucket); its other segment sums are rest[0 .. n_rest).  A bucket
// with more than kCombineSeq segments, and every bucket of a latency plan, is one point of `buckets`.
__device__ __forceinline__ g1_xyzz bucket_first(const TreeArgs& a, const g1_xyzz* buckets, size_t bk, const g1_xyzz*& rest,
                                                uint32_t& n_rest) {
    n_rest = 0;
    if (a.seg_offsets) {
        const uint32_t s0 = a.seg_offsets[bk], k = a.seg_offsets[bk + 1] - s0;
        if (k <= (uint32_t)kCombineSeq) {
            if (k == 0) return g1_xyzz_inf();
            rest = a.seg_sums + s0 + 1;
            n_rest = k - 1;
            return g1_xyzz_load(a.seg_sums + s0);
        }
    }
    return g1_xyzz_load(buckets + bk);
}

__global__ void __launch_bounds__(kTreeThreads) msm_tree_kernel(TreeArgs a) {
    const bool is_row = blockIdx.x < a.row.n_blocks;
    const TreeLevel& lv = is_row ? a.row : a.col;
    const uint32_t t = (is_row ? blockIdx.x : blockIdx.x - a.row.n_blocks) * kTreeThreads + threadIdx.x;
    if (t >= lv.n_out) return;
    const uint32_t inner_mask = (1u << lv.inner_log) - 1u;
    const size_t first = (((size_t)(t >> lv.inner_log) << lv.t_log) << lv.inner_log) | (t & inner_mask);
    const size_t stride = (size_t)1 << lv.inner_log;
    const uint32_t T = 1u << lv.t_log;
    // the points added, in order: bucket j's first segment sum, then its other ones, for j < T; the next one is fetched under
    // the addition of the current one
    const g1_xyzz* rest = nullptr;
    uint32_t n_rest, i = 0, j = 0;
    g1_xyzz acc = g1_xyzz_inf();
    g1_xyzz next = bucket_first(a, lv.in, first, rest, n_rest);
#pragma unroll 1
    while (true) {
        const g1_xyzz cur = next;
        bool more = true;
        if (i < n_rest) {
            next = g1_xyzz_load(rest + i++);
        } else if (++j < T) {
            next = bucket_first(a, lv.in, first + (size_t)j * stride, rest, n_rest);
            i = 0;
        } else {
            more = false;
        }
        acc = g1_add(acc, cur);
        if (!more) break;
    }
    g1_xyzz_store(lv.out + t, acc);
}

// The same level with four lanes per output (xyzz_add_quad): the chain of T - 1 additions is ~3x shorter and a quad's
// loads are one contiguous 128-byte point.  Per quad two shared-memory slots: the running sum and the next operand, whose
// successor is fetched (one coordinate per lane) under the addition.
template <int kThreads>
__global__ void __launch_bounds__(kThreads) msm_tree_quad_kernel(TreeArgs a) {
    __shared__ g1_xyzz sh[kThreads / 2];
    constexpr uint32_t kQuads = kThreads / 4;
    const bool is_row = blockIdx.x < a.row.n_blocks;
    const TreeLevel& lv = is_row ? a.row : a.col;
    const uint32_t blk = is_row ? blockIdx.x : blockIdx.x - a.row.n_blocks;
    const uint32_t ql = threadIdx.x >> 2, q = threadIdx.x & 3u;
    const uint32_t t = blk * kQuads + ql;
    const bool on = t < lv.n_out;
    if (__all_sync(0xffffffffu, !on)) return;  // a warp without outputs
    const uint32_t inner_mask = (1u << lv.inner_log) - 1u;
    const uint32_t tt = on ? t : 0u;
    const size_t first = (((size_t)(tt >> lv.inner_log) << lv.t_log) << lv.inner_log) | (tt & inner_mask);
    const size_t stride = (size_t)1 << lv.inner_log;
    const uint32_t T = 1u << lv.t_log;
    const fe* p = reinterpret_cast<const fe*>(lv.in + first) + q;  // coordinate q of the quad's inputs
    const size_t hop = stride * 4;                                 // in field elements
    fe* F = reinterpret_cast<fe*>(sh);
    const uint32_t sa = 2u * ql, sb = sa + 1u;
    fe_store(F + 4u * sa + q, fe_load(p));
    fe next = T > 1 ? fe_load(p + hop) : fe_zero();
#pragma unroll 1
    for (uint32_t j = 1; j < T; ++j) {
        fe_store(F + 4u * sb + q, next);
        __syncwarp();
        if (j + 1 < T) next = fe_load(p + (size_t)(j + 1) * hop);
        xyzz_add_quad(sh, sa, sb, on);
        __syncwarp();
    }
    __syncwarp();
    if (on) fe_store(reinterpret_cast<fe*>(lv.out + t) + q, fe_load(F + 4u * sa + q));
}

// Latency plans: second (and last) level of both trees: what the serial level leaves — 2^g partial sums per row / column, g <= 8 —
// is folded by a binary tree in shared memory, one addition per step on the critical path instead of 2^g - 1.
//   rows:    out[O] = sum_j in[O * G + j]                                  (G = 2^g partials of a row are contiguous)
//   columns: out[w * L + lo] = sum_j in[(w * G + j) * L + lo]             (the G partial rows of window w)
struct BlockTreePart {
    const g1_xyzz* in;
    g1_xyzz* out;
    uint32_t n_out, g_log, n_blocks;
};
struct BlockTreeArgs {
    BlockTreePart row, col;
    uint32_t l_log;
};
constexpr int kBlockTreeThreads = 256;

template <bool QUAD>
__global__ void __launch_bounds__(kBlockTreeThreads) msm_blocktree_kernel(BlockTreeArgs a) {
    __shared__ g1_xyzz sh[kBlockTreeThreads];
    const bool is_row = blockIdx.x < a.row.n_blocks;
    const BlockTreePart& p = is_row ? a.row : a.col;
    const uint32_t blk = is_row ? blockIdx.x : blockIdx.x - a.row.n_blocks;
    const uint32_t G = 1u << p.g_log, ob_log = 8u - p.g_log, OB = 1u << ob_log;  // outputs per block
    const uint32_t t = threadIdx.x;
    // rows: t = o * G + j (j fastest: contiguous loads); columns: t = j * OB + o (o fastest: adjacent columns)
    const uint32_t j = is_row ? (t & (G - 1u)) : (t >> ob_log);
    const uint32_t o = is_row ? (t >> p.g_log) : (t & (OB - 1u));
    const uint32_t O = blk * OB + o;
    const uint32_t hop = is_row ? 1u : OB;  // distance in `sh` between partials j and j + 1 of one output
    g1_xyzz v = g1_xyzz_inf();
    if (O < p.n_out) {
        size_t idx;
        if (is_row) {
            idx = ((size_t)O << p.g_log) | j;
        } else {
            const uint32_t w = O >> a.l_log, lo = O & ((1u << a.l_log) - 1u);
            idx = ((((size_t)w << p.g_log) | j) << a.l_log) | lo;
        }
        v = g1_xyzz_load(p.in + idx);
    }
    sh[t] = v;
    __syncthreads();
    // level s folds partial j + s into partial j (j < s): the writers of a level own slots nobody reads in it
#pragma unroll 1
    for (uint32_t s = G >> 1, s_log = p.g_log - 1u; s > 0; s >>= 1, --s_log) {
        const uint32_t pairs = OB * s;  // additions of this level
        if (!QUAD || pairs * 4u > (uint32_t)kBlockTreeThreads) {  // more additions than quads: one lane each
            if (j < s) {
                v = g1_add(v, sh[t + s * hop]);
                sh[t] = v;
            }
        } else if ((t & ~31u) < pairs * 4u) {  // warps with at least one addition; four lanes per addition
            const uint32_t pr = t >> 2;
            const bool on = pr < pairs;
            // rows: pair -> (o, j) = (pr / s, pr % s), slot o * G + j; columns: slot j * OB + o = pr
            const uint32_t ia = !on ? (uint32_t)kBlockTreeThreads - 1u : (is_row ? (((pr >> s_log) << p.g_log) | (pr & (s - 1u))) : pr);
            xyzz_add_quad(sh, ia, on ? ia + s * hop : ia, on);
        }
        __syncthreads();
    }
    if (j == 0 && O < p.n_out) g1_xyzz_store(p.out + O, QUAD ? sh[t] : v);
}

// Latency plans: what is left per window are the two weighted sums.  A dependent XYZZ addition costs a warp the latency of its
// chained field products whatever else the SM does, so this tail is arranged for the SHORTEST dependent chain, with
// every independent piece on its own SM:
//     L * sum_hi hi R[hi] + sum_lo (lo + 1) C[lo] = sum_b 2^b T_b,   b < c - 1,
//     T_b = sum of the C[lo] with bit b of (lo + 1) set  +  the R[hi] with bit (b - l) of hi set,
// msm_bitsum_kernel: one block per (window, bit) folds its <= L/2 (+ Rws/2) elements with a binary tree in
// shared memory (log2 steps of one addition each); msm_horner_kernel: one warp per window combines the c - 1
// bit sums pairwise — (T_b + 2 T_{b+1}), then (.. + 4 ..), (.. + 16 ..), ... — c - 2 doublings and
// ceil(log2(c - 1)) additions on the critical path instead of a scan over hundreds of elements.
constexpr int kBitThreads = 256;

template <bool QUAD>
__global__ void __launch_bounds__(kBitThreads) msm_bitsum_kernel(const g1_xyzz* __restrict__ col_sums, uint32_t l_log,
                                                                 const g1_xyzz* __restrict__ row_sums, uint32_t r_log,
                                                                 g1_xyzz* __restrict__ bit_sums /* [window][c - 1] */) {
    __shared__ g1_xyzz sh[kBitThreads];
    const uint32_t b = blockIdx.x, window = blockIdx.y, n_bits = gridDim.x;
    const g1_xyzz* C = col_sums + ((size_t)window << l_log);
    const g1_xyzz* R = row_sums + ((size_t)window << r_log);
    g1_xyzz acc = g1_xyzz_inf();
    uint32_t live = 1;  // threads 0 .. live - 1 may hold a point
    // column side: weights v = lo + 1 in [1, L]; bit b < l is set in L / 2 of them, bit l only in v = L
    if (b < l_log) {
        const uint32_t cnt = 1u << (l_log - 1), low_mask = (1u << b) - 1u;
        live = cnt;
#pragma unroll 1
        for (uint32_t j = threadIdx.x; j < cnt; j += kBitThreads) {
            const uint32_t v = ((j >> b) << (b + 1)) | (1u << b) | (j & low_mask);  // j-th value with bit b set
            acc = xyzz_add(acc, g1_xyzz_load(C + (v - 1u)));
        }
    } else if (b == l_log && threadIdx.x == 0) {
        acc = g1_xyzz_load(C + ((1u << l_log) - 1u));
    }
    // row side: weights hi * L, hi < Rws: bit b >= l of the weight is bit b - l of hi
    if (b >= l_log && r_log > 0) {
        const uint32_t rb = b - l_log, cnt = 1u << (r_log - 1), low_mask = (1u << rb) - 1u;
        live = cnt;
#pragma unroll 1
        for (uint32_t j = threadIdx.x; j < cnt; j += kBitThreads) {
            const uint32_t hi = ((j >> rb) << (rb + 1)) | (1u << rb) | (j & low_mask);
            acc = xyzz_add(acc, g1_xyzz_load(R + hi));
        }
    }
    sh[threadIdx.x] = acc;
    __syncthreads();
    // binary tree over the live slots (a power of two); the empty upper levels of the 256-slot tree are skipped
    uint32_t stride = kBitThreads / 2;
    if (QUAD) {
        if (live > (uint32_t)kBitThreads) live = kBitThreads;
        while (stride >= live && stride > 0) stride >>= 1;  // live = 1: nothing to fold
    }
#pragma unroll 1
    for (; stride > 0; stride >>= 1) {
        if (!QUAD || stride * 4u > (uint32_t)kBitThreads) {  // more additions than quads: one lane each
            if (threadIdx.x < stride) {
                acc = g1_add(acc, sh[threadIdx.x + stride]);
                sh[threadIdx.x] = acc;
            }
        } else if ((threadIdx.x & ~31u) < stride * 4u) {  // four lanes per addition
            const uint32_t pr = threadIdx.x >> 2;
            const bool on = pr < stride;
            xyzz_add_quad(sh, on ? pr : (uint32_t)kBitThreads - 1u, on ? pr + stride : (uint32_t)kBitThreads - 1u, on);
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) g1_xyzz_store(bit_sums + (size_t)window * n_bits + b, QUAD ? sh[0] : acc);
}

__device__ __forceinline__ g1_xyzz xyzz_shfl_down(const g1_xyzz& v, unsigned delta) {
    g1_xyzz r;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        r.x.l[k] = __shfl_down_sync(0xffffffffu, v.x.l[k], delta);
        r.y.l[k] = __shfl_down_sync(0xffffffffu, v.y.l[k], delta);
        r.zz.l[k] = __shfl_down_sync(0xffffffffu, v.zz.l[k], delta);
        r.zzz.l[k] = __shfl_down_sync(0xffffffffu, v.zzz.l[k], delta);
    }
    return r;
}

// window sum = sum_b 2^b T_b, n_bits <= 32: lane b starts with T_b; round s folds lane b + 2^s into lane b
// (b a multiple of 2^(s+1)) after 2^s doublings.
__global__ void __launch_bounds__(32) msm_horner_kernel(const g1_xyzz* __restrict__ bit_sums, uint32_t n_bits,
                                                        g1_xyzz* __restrict__ window_sums) {
    const uint32_t window = blockIdx.x, lane = threadIdx.x;
    g1_xyzz v = lane < n_bits ? g1_xyzz_load(bit_sums + (size_t)window * n_bits + lane) : g1_xyzz_inf();
#pragma unroll 1
    for (uint32_t s = 0; (1u << s) < n_bits; ++s) {
        g1_xyzz o = xyzz_shfl_down(v, 1u << s);
        if (lane + (1u << s) >= 32u) o = g1_xyzz_inf();
#pragma unroll 1
        for (uint32_t i = 0; i < (1u << s); ++i) o = g1_dbl(o);
        v = g1_add(v, o);
    }
    if (lane == 0) g1_xyzz_store(window_sums + window, v);
}

// ---- throughput plans: the reduction after the serial level as two wide levels of warp-local sums ------------------
// Both levels are many small independent sums, so they are laid out as throughput work: a sum of cnt points goes to a
// group of S = 2^s_log aligned lanes of one warp (rows / columns: S = cnt / 8, at least 4 and at most 32; bit sums: 32); lane k folds points
// k, k + S, ... one after the other and the group's lanes meet in log2(S) shuffle levels.  No shared memory, no block
// barrier, a few warps per block: the blocks hold an SM no longer than their own additions take.
//   msm_tail_kernel        R[O] and C[O] from the serial level's G = 2^g partials of row / column O
//   msm_tail_bits_kernel   the c - 1 bit sums T_b of each window from R and C (the weights of msm_bitsum_kernel)
constexpr int kTailThreads = 128;
constexpr uint32_t kTailFoldLog = 3;  // points folded one after the other by a lane before the shuffle levels

// log2 of the lanes that sum 2^cnt_log points: 2^cnt_log / 8, at least 4 (the small windows of small proofs: shorter
// chains, at c = 17 the same) and at most 32
constexpr uint32_t tail_group_log(uint32_t cnt_log) {
    return cnt_log <= 2u ? cnt_log : cnt_log <= kTailFoldLog + 2u ? 2u : cnt_log - kTailFoldLog < 5u ? cnt_log - kTailFoldLog : 5u;
}

// Sum of at(0) .. at(cnt - 1) by the group of 2^s_log lanes this lane is lane k of; the result is valid in lane k = 0.
// Every lane of the warp calls it (the shuffles are warp-wide): lanes with nothing to add pass cnt = 0.
template <class F>
__device__ __forceinline__ g1_xyzz group_sum(uint32_t k, uint32_t s_log, uint32_t cnt, F at) {
    const uint32_t S = 1u << s_log;
    g1_xyzz acc = g1_xyzz_inf();
    if (k < cnt) {
        g1_xyzz next = g1_xyzz_load(at(k));
#pragma unroll 1
        for (uint32_t i = k + S;; i += S) {
            const g1_xyzz cur = next;
            if (i < cnt) next = g1_xyzz_load(at(i));  // prefetch under the addition
            acc = xyzz_add(acc, cur);
            if (i >= cnt) break;
        }
    }
#pragma unroll 1
    for (uint32_t d = S >> 1; d > 0; d >>= 1) {
        g1_xyzz o = xyzz_shfl_down(acc, d);
        if (k >= d) o = g1_xyzz_inf();  // only lanes k < d carry on; the others must not pick up the next group's points
        acc = xyzz_add(acc, o);
    }
    return acc;
}

struct TailPart {
    const g1_xyzz* in;
    g1_xyzz* out;
    uint32_t n_out, g_log, s_log, n_warps;
};
struct TailArgs {
    TailPart row, col;
    uint32_t l_log;
};

//   rows:    R[O] = sum_j in[O * G + j]                        (G partials of a row are contiguous)
//   columns: C[w * L + lo] = sum_j in[(w * G + j) * L + lo]    (the G partial rows of window w)
__global__ void __launch_bounds__(kTailThreads) msm_tail_kernel(TailArgs a) {
    const uint32_t warp = (blockIdx.x * kTailThreads + threadIdx.x) >> 5, lane = threadIdx.x & 31u;
    if (warp >= a.row.n_warps + a.col.n_warps) return;  // whole warps
    const bool is_row = warp < a.row.n_warps;
    const TailPart& p = is_row ? a.row : a.col;
    const uint32_t idx = ((is_row ? warp : warp - a.row.n_warps) << 5) | lane;
    const uint32_t O = idx >> p.s_log, k = idx & ((1u << p.s_log) - 1u);
    const bool on = O < p.n_out;
    const uint32_t lo_mask = (1u << a.l_log) - 1u;
    const g1_xyzz sum = group_sum(k, p.s_log, on ? 1u << p.g_log : 0u, [&](uint32_t j) {
        return is_row ? p.in + (((size_t)O << p.g_log) | j)
                      : p.in + (((((size_t)(O >> a.l_log) << p.g_log) | j) << a.l_log) | (O & lo_mask));
    });
    if (on && k == 0) g1_xyzz_store(p.out + O, sum);
}

// bit_sums[w][b], b < c - 1 = l + r: T_b = the C[lo] of window w whose weight lo + 1 has bit b set, plus the R[hi] whose
// weight hi * L has bit b set (bit b - l of hi); bit l of lo + 1 is set only in lo + 1 = L.  One warp per bit sum.
__global__ void __launch_bounds__(kTailThreads) msm_tail_bits_kernel(const g1_xyzz* __restrict__ C, uint32_t l_log,
                                                                     const g1_xyzz* __restrict__ R, uint32_t r_log,
                                                                     uint32_t n_out, g1_xyzz* __restrict__ bit_sums) {
    const uint32_t O = (blockIdx.x * kTailThreads + threadIdx.x) >> 5, k = threadIdx.x & 31u;
    if (O >= n_out) return;  // whole warps
    const uint32_t n_bits = l_log + r_log, w = O / n_bits, b = O % n_bits;
    const g1_xyzz* Cw = C + ((size_t)w << l_log);
    const g1_xyzz* Rw = R + ((size_t)w << r_log);
    // column side (b < l): the j-th weight with bit b set is v = (j >> b) << (b + 1) | 1 << b | j mod 2^b, j < L / 2;
    // row side (b >= l): the same over hi with bit b - l, after C[L - 1] when b = l
    const uint32_t extra = b == l_log ? 1u : 0u;
    const uint32_t cnt = b < l_log ? 1u << (l_log - 1) : extra + (r_log ? 1u << (r_log - 1) : 0u);
    const uint32_t bb = b < l_log ? b : b - l_log, low_mask = (1u << bb) - 1u;
    const g1_xyzz sum = group_sum(k, 5u, cnt, [&](uint32_t j) {
        if (j < extra) return Cw + ((1u << l_log) - 1u);
        j -= extra;
        const uint32_t v = ((j >> bb) << (bb + 1)) | (1u << bb) | (j & low_mask);
        return b < l_log ? Cw + (v - 1u) : Rw + v;
    });
    if (k == 0) g1_xyzz_store(bit_sums + O, sum);
}

// ---- window tables: table[j][i] = 2^(shift*j) * P_i (affine) -------------------------------------
__global__ void msm_table_kernel(const g1_affine* __restrict__ prev, g1_affine* __restrict__ next,
                                 size_t n, int shift) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const g1_affine p = g1_affine_load_ro(prev + i);
    g1_xyzz a = g1_dbl_affine(p);
    for (int k = 1; k < shift; ++k) a = g1_dbl(a);
    g1_affine_store(next + i, g1_to_affine(a));
}

__global__ void g1_on_curve_kernel(const g1_affine* pts, size_t n, uint32_t* bad) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    if (!g1_affine_on_curve(g1_affine_load_ro(pts + i))) atomicAdd(bad, 1u);
}

// ---- synthetic inputs (SURVEY.md §8(d)): SplitMix64 field elements, known-dlog bases ---------------
__device__ __forceinline__ uint64_t splitmix_at(uint64_t seed, uint64_t j) {
    uint64_t z = seed + (j + 1) * 0x9E3779B97F4A7C15ULL;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ULL;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBULL;
    return z ^ (z >> 31);
}
__device__ __forceinline__ fe splitmix_fr_canon(uint64_t seed, uint64_t i) {
    fe v;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const uint64_t x = splitmix_at(seed, 4 * i + k);
        v.l[2 * k] = (uint32_t)x;
        v.l[2 * k + 1] = (uint32_t)(x >> 32);
    }
    // 2^256 / r < 6: a few conditional subtractions reduce mod r
    for (int it = 0; it < 6; ++it) {
        bool ge = true;
        for (int k = 7; k >= 0; --k) {
            if (v.l[k] != FrCfg::mod(k)) { ge = v.l[k] > FrCfg::mod(k); break; }
        }
        if (!ge) break;
        uint64_t borrow = 0;
        for (int k = 0; k < 8; ++k) {
            const uint64_t d = (uint64_t)v.l[k] - FrCfg::mod(k) - borrow;
            v.l[k] = (uint32_t)d;
            borrow = (d >> 32) & 1u;
        }
    }
    return v;
}
__global__ void splitmix_fr_kernel(uint64_t seed, size_t first, size_t n, int montgomery, fe* out) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    fe v = splitmix_fr_canon(seed, first + i);
    if (montgomery) v = fe_to_mont<FrCfg>(v);
    fe_store(out + i, v);
}
__global__ void known_dlog_bases_kernel(uint64_t seed, size_t first, size_t n, g1_affine* out) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const fe a = splitmix_fr_canon(seed, first + i);
    g1_affine g;
    g.x = fe_one<FqCfg>();
    g.y = fe_from_u32<FqCfg>(2);
    g1_affine_store(out + i, g1_to_affine(g1_mul_bits(g, a, 254)));
}

}  // namespace

// ---------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------
// c_override: 0 = choose for THROUGHPUT (many MSMs / proofs in flight on the GPU, the prover pool's regime: minimise the
// multiplier work), 1 = choose for LATENCY (one MSM at a time: minimise the dependent chains), >= 2 = that window.
MsmPlan msm_choose_plan(size_t n, int c_override, size_t mem_budget_bytes) {
    MsmPlan best;
    double best_cost = 1e300;
    const bool latency_mode = c_override == 1;
    const int c_lo = c_override > 1 ? c_override : 6, c_hi = c_override > 1 ? c_override : 23;
    for (int c = c_lo; c <= c_hi; ++c) {
        const int W = (255 + c - 1) / c;
        if (W > 32) continue;
        // Both models are in ms and were fitted to B200 measurements of these kernels; neither has been re-fitted on the
        // H100.  The throughput model's choice does not depend on the multiplier rate it divides by, so it carries over;
        // the latency model's constants are absolute B200 fits, kept unverified on the H100.
        // The top window of a 254-bit scalar has t = 254 - c (W - 1) bits: n entries pile into 2^t buckets there (hot
        // atomics in the sort; n / 2^t / 32 segments combined sequentially, up to 64, before the block-tree path).
        const int t = 254 - c * (W - 1);
        const double nw = (double)n * W;
        const int shrt = t >= c - 6 ? 0 : (c - 6 - t);
        double cost;
        if (!latency_mode) {
            // THROUGHPUT: Fq-product equivalents (divided by a fixed multiplier rate) — 9.5 per bucket addition, ~1.6 per digit for
            // the sort (more with a short top digit), 2 full additions (12.5 each) per bucket in the reduction.  With several proofs in flight this, not the chain length, is what a proof costs the GPU: at
            // n = 2^13 the latency-optimal c = 16 spends as much on reducing 2^15 buckets as on filling them.
            // Buckets with more than 32 entries are cut into segments whose sums are added up afterwards: with a Poisson
            // load of nw / buckets that is about max(0, load / 32 - 0.55) extra full additions per bucket (load 32 -> 0.45).
            // Checked against the pool at n = 2^16: c = 17 beats c = 16.
            const double buckets = (double)((size_t)1 << (c - 1));
            const double extra_segs = std::max(0.0, nw / 32.0 - 0.55 * buckets);
            cost = (nw * (9.5 + 1.6 * (1.0 + 0.3 * shrt)) + buckets * 25.0 + extra_segs * 12.5) / 66.7e6;
        } else {
            // LATENCY: a dependent curve addition costs a warp a long chain of multiplier-pipe time, so at the prover's sizes
            // every phase is a chain:
            //   sort        0.042 + n W / 54e6
            //   accumulate  max(throughput n W / 6.6e6,  chain 0.055 + 0.006 * min(load, 32) + 0.004 * segments) with
            //               load = n W / 2^(c-1) entries per bucket, cut into segments of 32
            //   reduce      0.13 + 0.0075 c (tree level, block tree, bit sums, pairwise Horner) + 2^c / 4.9e6
            const double load = nw / (double)((size_t)1 << (c - 1));
            const double segs = load / 32.0;
            const double acc = std::max(nw / 6.6e6, 0.055 + 0.006 * std::min(load, 32.0) + 0.004 * std::min(segs, 64.0));
            const double top_segs = t < c - 1 ? (double)n / (double)((size_t)1 << t) / 32.0 : 0.0;
            cost = 0.042 + nw * (1.0 + 0.1 * shrt) / 54e6 + acc + 0.13 + 0.0075 * c +
                   (double)((size_t)1 << c) / 4.9e6 + 0.008 * std::min(top_segs, 64.0);
        }
        if (cost < best_cost) {
            best_cost = cost;
            best.c = c;
            best.n_digits = W;
            best.latency = latency_mode ? 1 : 0;
        }
    }
    // full precompute (one physical window) unless the tables exceed the memory budget;
    // B200_MSM_PHYS_WINDOWS forces a split (tuning / test knob for the host Horner path)
    int phys = 1;
    if (const char* env = std::getenv("B200_MSM_PHYS_WINDOWS")) {
        const int v = std::atoi(env);
        if (v >= 1 && v <= best.n_digits) phys = v;
    }
    while (true) {
        const int tables = (best.n_digits + phys - 1) / phys;
        if ((double)tables * (double)n * 64.0 <= (double)mem_budget_bytes || phys >= best.n_digits) {
            best.n_phys = phys;
            best.n_tables = tables;
            break;
        }
        ++phys;
    }
    return best;
}

static int build_tables(Bases* b, cudaStream_t st) {
    const int shift = b->plan.c * b->plan.n_phys;
    const unsigned bs = 128;
    const unsigned grid = (unsigned)((b->n + bs - 1) / bs);
    for (int j = 1; j < b->plan.n_tables; ++j) {
        B200_LAUNCH(msm_table_kernel, grid, bs, 0, st)(b->tables + (size_t)(j - 1) * b->n,
                                              b->tables + (size_t)j * b->n, b->n, shift);
    }
    B200_CUDA(cudaGetLastError());
    B200_CUDA(cudaStreamSynchronize(st));
    return B200_OK;
}

static size_t table_mem_budget() {
    size_t free_b = 0, total_b = 0;
    if (cudaMemGetInfo(&free_b, &total_b) != cudaSuccess) return (size_t)8 << 30;
    return free_b / 2;
}

int bases_create_device(const g1_affine* d_points, size_t n, int c_override, cudaStream_t st,
                        Bases** out, size_t table_budget_bytes) {
    if (n == 0 || n > ((size_t)1 << kIdxBits)) {
        set_error("bases: n must be in [1, 2^26]");
        return B200_ERR_INVALID;
    }
    Bases* b = new Bases();
    b->n = n;
    b->plan = msm_choose_plan(n, c_override, table_budget_bytes == kTablesAuto ? table_mem_budget() : table_budget_bytes);
    cudaError_t e = cudaMalloc(&b->tables, (size_t)b->plan.n_tables * n * sizeof(g1_affine));
    if (e != cudaSuccess) {
        delete b;
        return cuda_fail(e, "cudaMalloc(window tables)");
    }
    e = cudaMemcpyAsync(b->tables, d_points, n * sizeof(g1_affine), cudaMemcpyDeviceToDevice, st);
    if (e != cudaSuccess) {
        delete b;
        return cuda_fail(e, "cudaMemcpyAsync(bases)");
    }
    int rc = build_tables(b, st);
    if (rc != B200_OK) {
        delete b;
        return rc;
    }
    *out = b;
    return B200_OK;
}

int bases_create(const g1_affine* h_points, size_t n, int c_override, int check_on_curve,
                 cudaStream_t st, Bases** out) {
    if (n == 0 || n > ((size_t)1 << kIdxBits)) {
        set_error("bases: n must be in [1, 2^26]");
        return B200_ERR_INVALID;
    }
    g1_affine* d_pts = nullptr;
    B200_CUDA(cudaMalloc(&d_pts, n * sizeof(g1_affine)));
    cudaError_t e = cudaMemcpyAsync(d_pts, h_points, n * sizeof(g1_affine), cudaMemcpyHostToDevice, st);
    if (e != cudaSuccess) {
        cudaFree(d_pts);
        return cuda_fail(e, "cudaMemcpyAsync(bases H2D)");
    }
    if (check_on_curve) {  // srs.rs:178-179 asserts every SRS point is on the curve
        uint32_t* d_bad = nullptr;
        uint32_t h_bad = 0;
        if ((e = cudaMalloc(&d_bad, 4)) != cudaSuccess) {
            cudaFree(d_pts);
            return cuda_fail(e, "cudaMalloc(on-curve flag)");
        }
        cudaMemsetAsync(d_bad, 0, 4, st);
        B200_LAUNCH(g1_on_curve_kernel, (unsigned)((n + 255) / 256), 256, 0, st)(d_pts, n, d_bad);
        cudaMemcpyAsync(&h_bad, d_bad, 4, cudaMemcpyDeviceToHost, st);
        e = cudaStreamSynchronize(st);
        cudaFree(d_bad);
        if (e != cudaSuccess) {
            cudaFree(d_pts);
            return cuda_fail(e, "on-curve check");
        }
        if (h_bad) {
            cudaFree(d_pts);
            set_error("point not on curve");
            return B200_ERR_NOT_ON_CURVE;
        }
    }
    int rc = bases_create_device(d_pts, n, c_override, st, out);
    cudaFree(d_pts);
    return rc;
}

// Bits of the column index (l) and of the row index (r), and how each tree splits them: `a` bits by the serial
// level (fan-in <= 8 per thread: the throughput part, two additions per bucket), the rest (<= 8 bits) by
// msm_tail_kernel (throughput plans) or the shared-memory binary tree of msm_blocktree_kernel (latency plans).
static void tree_shape(int c, int latency, size_t n_buckets, int* l_log, int* r_log, int* a_row, int* a_col) {
    const int bits = c - 1;
    const int l = (bits + 1) / 2, r = bits - l;
    *l_log = l;
    *r_log = r;
    // Fan-in 8 for the serial level, except in a latency plan with few buckets (one MSM alone up to c = 18; the 2^12
    // statement's batch of five): there fan-in 4 and one more quad level in the shared-memory tree is the shorter chain
    // (a shorter reduce of a lone 2^14 / 2^16-point MSM; with more buckets the doubled block-tree work costs more than the
    // chain saves).  No serial level at all was measured and lost, fan-in 2 loses everywhere above 2^13.
    // B200_TREE_FANIN_LOG = 1 | 2 | 3 forces the fan-in of latency plans (A/B measurements).
    static const int forced = [] {
        const char* e = std::getenv("B200_TREE_FANIN_LOG");
        return e && e[0] >= '1' && e[0] <= '3' ? e[0] - '0' : 0;
    }();
    int a = 3;
    if (latency) a = forced ? forced : (n_buckets <= kSmallTreeBuckets ? 2 : 3);
    if (l - a > 8) a = l - 8;  // the shared-memory tree takes at most 8 bits
    *a_row = l < a ? l : a;
    *a_col = r < a ? r : a;
}

// `batch` MSMs over the same bases (scalar vectors `stride` elements apart) in one pass: the
// digit sort, the bucket folding and the reduction each run once over batch * buckets buckets,
// which is what fills the GPU's SMs at the prover's 2^16-point sizes.
//
// msm_launch_batch only ENQUEUES (kernels + one D2H of the bit or window sums into pinned memory,
// as its MsmEpilogue says); msm_finish_batch waits for that copy and runs the host epilogue.  The
// prover queues further work between the two.
// B200_HOST_HORNER=0 keeps the last step of the reduction on the device (A/B measurements; read by msm_pending)
// B200_QUAD_ADD: 0 = one lane per addition everywhere (the round-1/2 kernels, kept for A/B measurements), 1 = four lanes per
// addition (xyzz_add_quad) in the two tail kernels, 2 (default) = and in the serial tree level of a latency plan with few outputs
static int quad_mode() {
    static const int mode = [] {
        const char* e = std::getenv("B200_QUAD_ADD");
        return e && e[0] >= '0' && e[0] <= '2' ? e[0] - '0' : 2;
    }();
    return mode;
}

MsmPending msm_pending(const Bases* b, size_t n, unsigned batch, MsmEpilogue e) {
    static const bool host_bits = [] {
        const char* v = std::getenv("B200_HOST_HORNER");
        return !(v && v[0] == '0');
    }();
    if (e == MsmEpilogue::HostBits && !host_bits) e = MsmEpilogue::HostWindows;
    return {b->plan, n, batch, e};
}

// sum_i t[i] 2^(shift i) over the n >= 1 terms, highest term first (Horner's rule)
static FF_HD g1_xyzz g1_horner_pow2(const g1_xyzz* t, int n, int shift) {
#ifdef __CUDA_ARCH__
    auto at = [&](int i) { return g1_xyzz_load(t + i); };  // 16-byte loads
#else
    auto at = [&](int i) { return t[i]; };
#endif
    g1_xyzz acc = at(n - 1);
    for (int i = n - 2; i >= 0; --i) {
        for (int k = 0; k < shift; ++k) acc = g1_dbl(acc);
        acc = g1_add(acc, at(i));
    }
    return acc;
}

// one MSM's window sums -> a single group element: Horner over the physical windows (a single window, the
// usual fully precomputed plan, passes through).  `empty`: the identity.
static __global__ void k_windows_to_point(const g1_xyzz* __restrict__ window_sums, int n_phys, int c, int empty,
                                          g1_xyzz* __restrict__ out) {
    if (threadIdx.x || blockIdx.x) return;
    if (empty) {
        g1_xyzz_store(out, g1_xyzz_inf());
        return;
    }
    g1_xyzz_store(out, g1_horner_pow2(window_sums, n_phys, c));
}

int msm_identity_point(g1_xyzz* d_point, cudaStream_t st) {
    B200_LAUNCH(k_windows_to_point, 1, 32, 0, st)(nullptr, 1, 1, 1, d_point);
    B200_CUDA(cudaGetLastError());
    return B200_OK;
}

// SMs the scratch's context may use: its partition's, or the current device's (132 on an H100 SXM).  The grid-stride
// heavy-bucket combine runs 4 blocks per SM.
static size_t sm_count(const MsmScratch* s) {
    if (s->sms) return s->sms;
    int dev = 0, sms = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess ||
        sms <= 0)
        return 132;
    return (size_t)sms;
}

size_t msm_scratch_estimate(const MsmPlan& pl, size_t points, size_t batch) {
    const size_t n_buckets = (size_t)pl.n_phys * ((size_t)1 << (pl.c - 1)) * batch;
    const size_t n_windows = (size_t)pl.n_phys * batch;
    const size_t entries = points * (size_t)pl.n_digits * batch;
    const size_t segs = entries / kSegLen + n_buckets;
    const size_t heavy = segs / (kCombineSeq + 1) + 2;
    const int l_log = pl.c / 2;
    const size_t tree = (n_buckets >> 1) + n_windows * (((size_t)1 << l_log) + ((size_t)1 << (pl.c - 1 - l_log))) + 1;
    return 4 * (5 * n_buckets + 2) + 4 * entries + (sizeof(g1_xyzz) + 8) * segs + 4 * segs + 4 * heavy +
           sizeof(g1_xyzz) * (tree + 65 * n_windows) + 4096;
}

int msm_launch_batch(const Bases* b, size_t base_off, const fe* d_scalars, size_t n, size_t stride, unsigned batch,
                     int montgomery, MsmEpilogue epilogue, MsmScratch* s, cudaStream_t st, MsmPending* pending,
                     g1_xyzz* d_point) {
    if (base_off + n > b->n) {
        set_error("msm: base_off + n exceeds the loaded bases");
        return B200_ERR_INVALID;
    }
    *pending = msm_pending(b, n, batch, epilogue);
    if (batch == 0 || n == 0) return B200_OK;
    const MsmPlan& pl = b->plan;
    const uint32_t half = 1u << (pl.c - 1);
    const size_t buckets_per_msm = (size_t)pl.n_phys * half;
    const size_t n_buckets = buckets_per_msm * batch;
    const size_t n_windows = (size_t)pl.n_phys * batch;
    const size_t max_entries = n * (size_t)pl.n_digits * batch;
    // segments: at most floor(entries / kSegLen) full ones plus one partial per bucket
    const size_t max_segs = max_entries / kSegLen + n_buckets;
    if (max_entries >= ((size_t)1 << 32) || n_buckets >= ((size_t)1 << 31) || max_segs >= ((size_t)1 << 30)) {
        set_error("msm: batch * n * windows exceeds the 2^32-entry / 2^30-segment index space");
        return B200_ERR_INVALID;
    }
    int rc;
    const size_t n_tiles = (n_buckets + kScanTile - 1) / kScanTile;
    if (s->counts.cap < n_buckets * 4) {  // a fresh histogram starts zeroed; every MSM leaves it zeroed
        if ((rc = s->counts.reserve(n_buckets * 4)) != B200_OK) return rc;
        B200_CUDA(cudaMemsetAsync(s->counts.p, 0, s->counts.cap, st));
    }
    if (s->scan_state.cap < sizeof(ScanState) + n_tiles * 8) {
        if ((rc = s->scan_state.reserve(sizeof(ScanState) + n_tiles * 8 + 1024)) != B200_OK) return rc;
        B200_CUDA(cudaMemsetAsync(s->scan_state.p, 0, s->scan_state.cap, st));
    }
    if ((rc = s->offsets.reserve((n_buckets + 1) * 4)) != B200_OK) return rc;
    if ((rc = s->cursor.reserve(n_buckets * 4)) != B200_OK) return rc;
    if ((rc = s->entries.reserve(max_entries * 4)) != B200_OK) return rc;
    if ((rc = s->buckets.reserve(n_buckets * sizeof(g1_xyzz))) != B200_OK) return rc;
    const size_t max_heavy = max_segs / (kCombineSeq + 1) + 1;
    if ((rc = s->seg_offsets.reserve((n_buckets + 1) * 4)) != B200_OK) return rc;
    if ((rc = s->seg_bucket.reserve(max_segs * 4)) != B200_OK) return rc;
    if ((rc = s->seg_sums.reserve(max_segs * sizeof(g1_xyzz))) != B200_OK) return rc;
    if ((rc = s->heavy.reserve((max_heavy + 1) * 4)) != B200_OK) return rc;
    if ((rc = s->seg_order.reserve(max_segs * 4)) != B200_OK) return rc;
    int l_log, r_log, a_row, a_col;
    tree_shape(pl.c, pl.latency, n_buckets, &l_log, &r_log, &a_row, &a_col);
    if (l_log - a_row > 8 || r_log - a_col > 8) {
        set_error("msm: window too wide for the two-level bucket reduction");
        return B200_ERR_INVALID;
    }
    // tree outputs: the serial level's partials, then the row sums R and column sums C
    const size_t row_l1 = n_buckets >> a_row, col_l1 = n_buckets >> a_col;
    const size_t n_R = n_windows << r_log, n_C = n_windows << l_log;
    const size_t tree_elems = row_l1 + col_l1 + n_R + n_C;
    if ((rc = s->tree.reserve((tree_elems + 1) * sizeof(g1_xyzz))) != B200_OK) return rc;
    if ((rc = s->window_sums.reserve(n_windows * sizeof(g1_xyzz))) != B200_OK) return rc;
    if ((rc = s->h_sums.reserve(n_windows * 32 * sizeof(g1_xyzz))) != B200_OK) return rc;  // window sums, or their c - 1 bit sums
    if (!s->done_ev) B200_CUDA(cudaEventCreateWithFlags(&s->done_ev, cudaEventDisableTiming));
    if ((rc = s->bit_sums.reserve(n_windows * 32 * sizeof(g1_xyzz))) != B200_OK) return rc;

    uint32_t* counts = (uint32_t*)s->counts.p;
    uint32_t* offsets = (uint32_t*)s->offsets.p;
    uint32_t* cursor = (uint32_t*)s->cursor.p;
    uint32_t* entries = (uint32_t*)s->entries.p;
    g1_xyzz* buckets = (g1_xyzz*)s->buckets.p;
    g1_xyzz* window_sums = (g1_xyzz*)s->window_sums.p;
    uint32_t* seg_offsets = (uint32_t*)s->seg_offsets.p;
    uint32_t* seg_bucket = (uint32_t*)s->seg_bucket.p;
    g1_xyzz* seg_sums = (g1_xyzz*)s->seg_sums.p;
    ScanState* stt = (ScanState*)s->scan_state.p;
    uint64_t* status = (uint64_t*)((char*)s->scan_state.p + sizeof(ScanState));
    uint32_t* heavy_list = (uint32_t*)s->heavy.p;
    uint32_t* seg_order = (uint32_t*)s->seg_order.p;

    cudaStreamCaptureStatus capture = cudaStreamCaptureStatusNone;
    B200_CUDA(cudaStreamIsCapturing(st, &capture));
    const bool capturing = capture != cudaStreamCaptureStatusNone;
    const bool timing = s->timing;
    if (timing && !s->ev_init) {
        for (auto& e : s->ev) B200_CUDA(cudaEventCreate(&e));
        s->ev_init = true;
    }
    // inside a stream capture a timing event has to become a node of the graph (external record), or a replay would not record it
    auto stamp = [&](int i) {
        if (!timing) return;
        if (capturing) cudaEventRecordWithFlags(s->ev[i], st, cudaEventRecordExternal);
        else cudaEventRecord(s->ev[i], st);
    };
    stamp(0);
    const unsigned bs = 256;
    const dim3 grid_n((unsigned)((n + bs - 1) / bs), batch);
    B200_LAUNCH(msm_count_kernel, grid_n, bs, 0, st)(d_scalars, n, stride, montgomery, pl, (uint32_t)buckets_per_msm, counts);
    B200_LAUNCH(msm_scan_kernel, (unsigned)n_tiles, kScanThreads, 0, st)(counts, (uint32_t)n_buckets, (uint32_t)n_tiles, stt, status,
                                                                offsets, cursor, seg_offsets);
    B200_LAUNCH(msm_scatter_kernel, grid_n, bs, 0, st)(d_scalars, n, stride, montgomery, pl, (uint32_t)base_off,
                                              (uint32_t)buckets_per_msm, cursor, entries);
    B200_LAUNCH(msm_segorder_kernel, (unsigned)((n_buckets + 255) / 256), 256, 0, st)(offsets, seg_offsets, (uint32_t)n_buckets,
                                                                             stt->seg_starts, seg_bucket, seg_order,
                                                                             &stt->heavy_count, heavy_list);
    // the long kernels of the MSM go to the low-priority companion stream (see b200_init)
    cudaStream_t hv = s->hv_stream ? s->hv_stream : st;
    stamp(1);
    if (s->hv_stream) {
        cudaEventRecord(s->hv_fork, st);
        cudaStreamWaitEvent(hv, s->hv_fork, 0);
    }
    B200_LAUNCH(msm_accumulate_kernel, (unsigned)((max_segs + 127) / 128), 128, 0, hv)(
        entries, offsets, seg_offsets, seg_bucket, seg_order, b->tables, b->n, (uint32_t)n_buckets, seg_sums);
    if (s->hv_stream) {
        cudaEventRecord(s->hv_join, hv);
        cudaStreamWaitEvent(st, s->hv_join, 0);
    }
    if (pl.latency)
        B200_LAUNCH(msm_bucket_combine_kernel, (unsigned)((n_buckets + 127) / 128), 128, 0, st)(seg_sums, seg_offsets,
                                                                                              (uint32_t)n_buckets, buckets);
    B200_LAUNCH(msm_heavy_combine_kernel, (unsigned)std::min<size_t>(max_heavy, 4 * sm_count(s)), kReduceThreads, 0, st)(
        seg_sums, seg_offsets, &stt->heavy_count, heavy_list, buckets);
    stamp(2);
    const unsigned n_bits = (unsigned)(pl.c - 1);
    g1_xyzz* bit_sums = (g1_xyzz*)s->bit_sums.p;
    g1_xyzz* t0 = (g1_xyzz*)s->tree.p;
    g1_xyzz *row_p = t0, *col_p = t0 + row_l1, *R = col_p + col_l1, *Cs = R + n_R;
    if (!pl.latency) {
        // serial level over the segment sums (both sides even at fan-in 1: nothing else reads the buckets), then the two
        // warp-sum levels of msm_tail_kernel / msm_tail_bits_kernel
        TreeArgs a;
        a.row = TreeLevel{buckets, row_p, (uint32_t)row_l1, (uint32_t)a_row, 0, 0};
        a.col = TreeLevel{buckets, col_p, (uint32_t)col_l1, (uint32_t)a_col, (uint32_t)l_log, 0};
        a.row.n_blocks = (a.row.n_out + kTreeThreads - 1) / kTreeThreads;
        a.col.n_blocks = (a.col.n_out + kTreeThreads - 1) / kTreeThreads;
        a.seg_offsets = seg_offsets;
        a.seg_sums = seg_sums;
        B200_LAUNCH(msm_tree_kernel, a.row.n_blocks + a.col.n_blocks, kTreeThreads, 0, st)(a);
        TailArgs ta;
        ta.l_log = (uint32_t)l_log;
        const uint32_t gr = (uint32_t)(l_log - a_row), gc = (uint32_t)(r_log - a_col);
        ta.row = TailPart{row_p, R, (uint32_t)n_R, gr, 0, 0};
        ta.col = TailPart{col_p, Cs, (uint32_t)n_C, gc, 0, 0};
        for (TailPart* p : {&ta.row, &ta.col}) {
            p->s_log = tail_group_log(p->g_log);
            p->n_warps = (uint32_t)((((size_t)p->n_out << p->s_log) + 31) / 32);
        }
        const uint32_t tail_warps = ta.row.n_warps + ta.col.n_warps;
        B200_LAUNCH(msm_tail_kernel, (tail_warps * 32 + kTailThreads - 1) / kTailThreads, kTailThreads, 0, st)(ta);
        // c - 1 bit sums per window are too few to fill the GPU and end a lone MSM's chain: a whole warp each
        const uint32_t n_out = (uint32_t)(n_windows * n_bits);
        B200_LAUNCH(msm_tail_bits_kernel, (n_out * 32 + kTailThreads - 1) / kTailThreads, kTailThreads, 0, st)(
            Cs, (uint32_t)l_log, R, (uint32_t)r_log, n_out, bit_sums);
    } else {
        const bool quad = quad_mode() >= 1;
        const g1_xyzz *row_in = buckets, *col_in = buckets;
        if (a_row || a_col) {  // serial level: out[a * inner + b] = sum_{j < 2^a} in[(a * 2^a + j) * inner + b]
            TreeArgs a;
            a.row = TreeLevel{buckets, row_p, a_row ? (uint32_t)row_l1 : 0u, (uint32_t)a_row, 0, 0};
            a.col = TreeLevel{buckets, col_p, a_col ? (uint32_t)col_l1 : 0u, (uint32_t)a_col, (uint32_t)l_log, 0};
            a.seg_offsets = nullptr;
            a.seg_sums = nullptr;
            a.row.n_blocks = (a.row.n_out + kTreeThreads - 1) / kTreeThreads;
            a.col.n_blocks = (a.col.n_out + kTreeThreads - 1) / kTreeThreads;
            // four lanes per output only where the level is a latency chain: a latency plan (one MSM alone) with fewer outputs
            // than the machine has lanes.  As throughput work the quad form just adds its exchange overhead: used everywhere
            // it slowed the 2^20-point MSM's reduce and the headline, and with the size rule alone the pool's small
            // statements were slower than with the tail kernels only
            if (quad_mode() >= 2 && (size_t)a.row.n_out + a.col.n_out <= kQuadTreeMaxOutputs) {
                constexpr unsigned kQ = kTreeThreads / 4;  // outputs per block
                a.row.n_blocks = (a.row.n_out + kQ - 1) / kQ;
                a.col.n_blocks = (a.col.n_out + kQ - 1) / kQ;
                B200_LAUNCH(msm_tree_quad_kernel<kTreeThreads>, a.row.n_blocks + a.col.n_blocks, kTreeThreads, 0, st)(a);
            } else {
                B200_LAUNCH(msm_tree_kernel, a.row.n_blocks + a.col.n_blocks, kTreeThreads, 0, st)(a);
            }
            if (a_row) row_in = row_p;
            if (a_col) col_in = col_p;
        }
        {   // binary trees over what is left of each row / column
            const int gr = l_log - a_row, gc = r_log - a_col;
            BlockTreeArgs a;
            a.l_log = (uint32_t)l_log;
            a.row = BlockTreePart{row_in, R, gr ? (uint32_t)n_R : 0u, (uint32_t)gr, 0};
            a.col = BlockTreePart{col_in, Cs, gc ? (uint32_t)n_C : 0u, (uint32_t)gc, 0};
            a.row.n_blocks = gr ? (uint32_t)((n_R + (256u >> gr) - 1) / (256u >> gr)) : 0u;
            a.col.n_blocks = gc ? (uint32_t)((n_C + (256u >> gc) - 1) / (256u >> gc)) : 0u;
            if (a.row.n_blocks + a.col.n_blocks)
                if (quad) B200_LAUNCH(msm_blocktree_kernel<true>, a.row.n_blocks + a.col.n_blocks, kBlockTreeThreads, 0, st)(a);
                else B200_LAUNCH(msm_blocktree_kernel<false>, a.row.n_blocks + a.col.n_blocks, kBlockTreeThreads, 0, st)(a);
            if (gr) row_in = R;
            if (gc) col_in = Cs;
        }
        // row_in: R[window][2^r_log], col_in: C[window][2^l_log]
        if (quad) B200_LAUNCH(msm_bitsum_kernel<true>, dim3(n_bits, (unsigned)n_windows), kBitThreads, 0, st)(col_in, (uint32_t)l_log, row_in,
                                                                                                     (uint32_t)r_log, bit_sums);
        else B200_LAUNCH(msm_bitsum_kernel<false>, dim3(n_bits, (unsigned)n_windows), kBitThreads, 0, st)(col_in, (uint32_t)l_log, row_in,
                                                                                                      (uint32_t)r_log, bit_sums);
    }
    // The last step, sum_b 2^b T_b, is a chain of c - 2 dependent doublings whoever runs it, and a host core runs it an
    // order of magnitude faster than a lone warp.  The host takes it (msm_finish_batch) unless the epilogue says otherwise.
    const MsmEpilogue e = pending->epilogue;
    if (e != MsmEpilogue::HostBits) B200_LAUNCH(msm_horner_kernel, (unsigned)n_windows, 32, 0, st)(bit_sums, n_bits, window_sums);
    if (e == MsmEpilogue::DevicePoint) B200_LAUNCH(k_windows_to_point, 1, 32, 0, st)(window_sums, pl.n_phys, pl.c, 0, d_point);
    B200_CUDA(cudaGetLastError());
    stamp(3);
    if (e == MsmEpilogue::HostBits)
        B200_CUDA(cudaMemcpyAsync(s->h_sums.p, s->bit_sums.p, n_windows * (size_t)(pl.c - 1) * sizeof(g1_xyzz), cudaMemcpyDeviceToHost, st));
    else if (e == MsmEpilogue::HostWindows)
        B200_CUDA(cudaMemcpyAsync(s->h_sums.p, window_sums, n_windows * sizeof(g1_xyzz), cudaMemcpyDeviceToHost, st));
    stamp(4);
    if (!capturing) B200_CUDA(cudaEventRecord(s->done_ev, st));  // a replaying caller records it after the graph launch
    return B200_OK;
}

// phase times of the MSM whose events have completed (the caller has waited for the stream / done_ev)
void msm_collect_timing(MsmScratch* s, size_t n, unsigned batch) {
    if (!s->timing || !s->ev_init) return;
    cudaEventElapsedTime(&s->ms[0], s->ev[0], s->ev[4]);
    cudaEventElapsedTime(&s->ms[1], s->ev[0], s->ev[1]);
    cudaEventElapsedTime(&s->ms[2], s->ev[1], s->ev[2]);
    cudaEventElapsedTime(&s->ms[3], s->ev[2], s->ev[3]);
    s->tot_acc_ms += s->ms[2];
    s->tot_pairs += (double)n * batch;
    s->tot_launches += 1;
}

int msm_finish_batch(MsmScratch* s, const MsmPending& p, g1_affine* out, int* out_inf) {
    const unsigned batch = p.batch;
    if (batch == 0) return B200_OK;
    if (p.n == 0) {
        for (unsigned i = 0; i < batch; ++i) {
            out[i].x = fe_zero();
            out[i].y = fe_zero();
            if (out_inf) out_inf[i] = 1;
        }
        return B200_OK;
    }
    const MsmPlan& pl = p.plan;
    B200_CUDA(cudaEventSynchronize(s->done_ev));
    msm_collect_timing(s, p.n, batch);
    // host epilogue: per MSM a Horner over the physical windows (none when fully precomputed), then
    // ONE field inversion for the whole batch (Montgomery's trick over the ZZZ coordinates) — a few
    // hundred bytes of work, read straight from the pinned copy of the window sums.
    const g1_xyzz* h_sums = reinterpret_cast<const g1_xyzz*>(s->h_sums.p);
    std::vector<g1_xyzz> wsum;
    if (p.epilogue == MsmEpilogue::HostBits) {  // window sum = sum_b 2^b T_b from the c - 1 bit sums of each window
        const int n_bits = pl.c - 1;
        wsum.resize((size_t)batch * pl.n_phys);
        for (size_t w = 0; w < wsum.size(); ++w) wsum[w] = g1_horner_pow2(h_sums + w * (size_t)n_bits, n_bits, 1);
        h_sums = wsum.data();
    }
    std::vector<g1_xyzz> totals(batch);
    std::vector<fe> prefix(batch);
    fe run = fe_one<FqCfg>();
    for (unsigned i = 0; i < batch; ++i) {
        const g1_xyzz total = g1_horner_pow2(h_sums + (size_t)i * pl.n_phys, pl.n_phys, pl.c);
        totals[i] = total;
        prefix[i] = run;
        if (!g1_xyzz_is_inf(total)) run = fe_mul<FqCfg>(run, total.zzz);
    }
    fe inv = fe_inv<FqCfg>(run);
    for (unsigned i = batch; i-- > 0;) {
        const g1_xyzz& t = totals[i];
        if (g1_xyzz_is_inf(t)) {
            out[i].x = fe_zero();
            out[i].y = fe_zero();
            if (out_inf) out_inf[i] = 1;
            continue;
        }
        const fe i3 = fe_mul<FqCfg>(inv, prefix[i]);  // 1 / ZZZ_i
        inv = fe_mul<FqCfg>(inv, t.zzz);
        const fe izz = fe_mul<FqCfg>(fe_sqr<FqCfg>(t.zz), fe_sqr<FqCfg>(i3));  // 1/ZZ = ZZ^2 / ZZZ^2
        out[i].x = fe_mul<FqCfg>(t.x, izz);
        out[i].y = fe_mul<FqCfg>(t.y, i3);
        if (out_inf) out_inf[i] = 0;
    }
    return B200_OK;
}

int msm_device_batch(const Bases* b, size_t base_off, const fe* d_scalars, size_t n, size_t stride,
                     unsigned batch, int montgomery, MsmScratch* s, cudaStream_t st, g1_affine* out,
                     int* out_inf) {
    MsmPending p;
    const int rc = msm_launch_batch(b, base_off, d_scalars, n, stride, batch, montgomery, MsmEpilogue::HostBits, s, st, &p);
    if (rc != B200_OK) return rc;
    return msm_finish_batch(s, p, out, out_inf);
}

int msm_device(const Bases* b, size_t base_off, const fe* d_scalars, size_t n, int montgomery,
               MsmScratch* s, cudaStream_t st, g1_affine* out, int* out_inf) {
    return msm_device_batch(b, base_off, d_scalars, n, n, 1, montgomery, s, st, out, out_inf);
}

int g1_known_dlog_bases_device(uint64_t seed, size_t first, size_t n, g1_affine* d_out,
                               cudaStream_t st) {
    if (n == 0) return B200_OK;
    B200_LAUNCH(known_dlog_bases_kernel, (unsigned)((n + 127) / 128), 128, 0, st)(seed, first, n, d_out);
    B200_CUDA(cudaGetLastError());
    return B200_OK;
}

int splitmix_fr_device(uint64_t seed, size_t first, size_t n, int montgomery, fe* d_out,
                       cudaStream_t st) {
    if (n == 0) return B200_OK;
    B200_LAUNCH(splitmix_fr_kernel, (unsigned)((n + 255) / 256), 256, 0, st)(seed, first, n, montgomery, d_out);
    B200_CUDA(cudaGetLastError());
    return B200_OK;
}

}  // namespace b200
