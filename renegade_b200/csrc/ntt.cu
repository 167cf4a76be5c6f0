// Radix-2 NTT / iNTT over the BN254 scalar field for sm_90a.
//
// Replaces what the reference reaches through ark-poly 0.4.2
// `Radix2EvaluationDomain::<Fr>::{fft, ifft, coset_fft, coset_ifft}` (called from the upstream
// prover behind /root/reference/crates/circuits/circuit-types/src/traits.rs:850,996; semantics
// restated in SURVEY.md App. B): natural order in, natural order out, ifft scales by n^-1,
// coset shift g = Fr::GENERATOR = 5.  Outputs are canonical field elements, so a correct NTT
// is bit-identical to arkworks'.
//
// Structure (device-first, not a translation of arkworks' recursive CPU FFT):
//   * decimation-in-frequency, log n stages grouped into ceil(log n / 10) passes; a pass keeps
//     a tile of 1024 elements (32 KB, two 128-bit planes to stay bank-conflict free) in shared
//     memory, so HBM sees one read + one write of the vector per pass;
//   * one element is one 32-byte sector, so the strided tile gathers of the upper passes and
//     the bit-reversed scatter of the last pass are all full-sector transactions;
//   * twiddles come from an L2-resident table (n/2 elements per direction); coset scaling and
//     the n^-1 factor are fused into the first load / last store.
// The kernel is bound by the integer-multiply pipe (≈ log2(n)/2 Montgomery products per
// element), not by HBM: see DESIGN.md for the roofline.
#include <cstdlib>

#include "device_ctx.h"
#include "ff.cuh"

namespace b200 {

namespace {

#ifndef B200_NTT_TILE_LOG
#define B200_NTT_TILE_LOG 10
#endif
constexpr int kTileLog = B200_NTT_TILE_LOG;  // 1024 elements = 32 KB of shared memory per block

struct PassArgs {
    const fe* in;
    fe* out;
    const fe* tw;     // w^k, k < n/2 (forward or inverse roots)
    const fe* pre;    // optional per-input-index factor (coset_fft: g^i)
    const fe* post;   // optional per-output-index factor (coset_ifft: g^-i * n^-1)
    fe post_scalar;   // used when has_post_scalar (ifft: n^-1)
    int has_post_scalar;
    int log_n, lo, hi;  // this pass runs butterfly stages hi-1 .. lo
    int e_log;          // tile = 2^e_log elements
    size_t batch_stride;  // elements between consecutive transforms of a batch
};

struct TileGeom {
    int E, t_log, q_log;
    uint32_t T_mask, Q_mask, lo_mask;
};
__device__ __forceinline__ TileGeom tile_geom(const PassArgs& a) {
    TileGeom g;
    g.E = 1 << a.e_log;
    g.t_log = a.hi - a.lo;              // sub-transform size 2^t_log
    g.q_log = a.e_log - g.t_log;        // sub-transforms per tile
    g.T_mask = (1u << g.t_log) - 1u;
    g.Q_mask = (1u << g.q_log) - 1u;
    g.lo_mask = (1u << a.lo) - 1u;
    return g;
}
// element e of the tile starting at sub-transform q_base: its index in the vector and its slot in shared memory
__device__ __forceinline__ void tile_slot(const PassArgs& a, const TileGeom& g, uint32_t q_base, uint32_t e, size_t* idx, uint32_t* pos) {
    uint32_t qq, m;
    if (a.lo == 0) { qq = e >> g.t_log; m = e & g.T_mask; }   // idx = q*T + m : contiguous in e
    else           { m = e >> g.q_log; qq = e & g.Q_mask; }   // adjacent sub-transforms adjacent
    const uint32_t q = q_base + qq;
    *idx = ((size_t)(q >> a.lo) << a.hi) | ((size_t)m << a.lo) | (q & g.lo_mask);
    *pos = (m << g.q_log) | qq;
}

// butterfly stages of this pass on the tile held in (plane_lo, plane_hi), then the scatter to `out`
template <bool FINAL>
__device__ __forceinline__ void tile_compute(const PassArgs& a, const TileGeom& g, uint4* plane_lo, uint4* plane_hi, uint32_t q_base,
                                             fe* out) {
    const int E = g.E, t_log = g.t_log, q_log = g.q_log;
    const uint32_t T_mask = g.T_mask, Q_mask = g.Q_mask, lo_mask = g.lo_mask;
    (void)T_mask;
    // ---- butterflies, two stages per shared-memory round trip (radix 4 in registers) ----------
    // stage s pairs indices 2^s apart: (x0, x1) -> (x0 + x1, (x0 - x1) * w^(j * n / 2^(s+1))), j = idx mod 2^s.
    auto lds = [&](uint32_t pos) {
        const uint4 u = plane_lo[pos], v = plane_hi[pos];
        fe x;
        x.l[0] = u.x; x.l[1] = u.y; x.l[2] = u.z; x.l[3] = u.w;
        x.l[4] = v.x; x.l[5] = v.y; x.l[6] = v.z; x.l[7] = v.w;
        return x;
    };
    auto sts = [&](uint32_t pos, const fe& y) {
        plane_lo[pos] = make_uint4(y.l[0], y.l[1], y.l[2], y.l[3]);
        plane_hi[pos] = make_uint4(y.l[4], y.l[5], y.l[6], y.l[7]);
    };
    int sp = t_log - 1;
    // the last pass ends on stages 1 and 0, whose twiddles are 1, 1, w^(n/4), 1: peeled below without the
    // three trivial products
    for (; sp >= 2 || (!FINAL && sp == 1); sp -= 2) {
        const int s = a.lo + sp;
        const uint32_t low_mask = (1u << (sp - 1)) - 1u;
        for (uint32_t t = threadIdx.x; t < (uint32_t)(E >> 2); t += blockDim.x) {
            const uint32_t qq = t & Q_mask;
            const uint32_t r = t >> q_log;
            const uint32_t low = r & low_mask;
            const uint32_t base = ((r >> (sp - 1)) << (sp + 1)) | low;
            const uint32_t lw = (q_base + qq) & lo_mask;
            const uint32_t p00 = (base << q_log) | qq;
            const uint32_t p01 = ((base | (1u << (sp - 1))) << q_log) | qq;
            const uint32_t p10 = ((base | (1u << sp)) << q_log) | qq;
            const uint32_t p11 = ((base | (3u << (sp - 1))) << q_log) | qq;
            const size_t j0 = ((size_t)low << a.lo) | lw;
            const size_t j1 = ((size_t)(low | (1u << (sp - 1))) << a.lo) | lw;
            const fe w0 = fe_load_ro(a.tw + (j0 << (a.log_n - s - 1)));
            const fe w1 = fe_load_ro(a.tw + (j1 << (a.log_n - s - 1)));
            const fe wp = fe_load_ro(a.tw + (j0 << (a.log_n - s)));
            const fe x00 = lds(p00), x01 = lds(p01), x10 = lds(p10), x11 = lds(p11);
            const fe y00 = fe_add<FrCfg>(x00, x10);
            const fe y10 = fe_mul<FrCfg>(fe_sub<FrCfg>(x00, x10), w0);
            const fe y01 = fe_add<FrCfg>(x01, x11);
            const fe y11 = fe_mul<FrCfg>(fe_sub<FrCfg>(x01, x11), w1);
            sts(p00, fe_add<FrCfg>(y00, y01));
            sts(p01, fe_mul<FrCfg>(fe_sub<FrCfg>(y00, y01), wp));
            sts(p10, fe_add<FrCfg>(y10, y11));
            sts(p11, fe_mul<FrCfg>(fe_sub<FrCfg>(y10, y11), wp));
        }
        __syncthreads();
    }
    if (FINAL && sp == 1) {
        const fe wi = fe_load_ro(a.tw + ((size_t)1 << (a.log_n - 2)));  // primitive 4th root (or its inverse)
        for (uint32_t t = threadIdx.x; t < (uint32_t)(E >> 2); t += blockDim.x) {
            const uint32_t qq = t & Q_mask;
            const uint32_t base = (t >> q_log) << 2;
            const uint32_t p00 = (base << q_log) | qq, p01 = ((base | 1u) << q_log) | qq;
            const uint32_t p10 = ((base | 2u) << q_log) | qq, p11 = ((base | 3u) << q_log) | qq;
            const fe x00 = lds(p00), x01 = lds(p01), x10 = lds(p10), x11 = lds(p11);
            const fe y00 = fe_add<FrCfg>(x00, x10), y10 = fe_sub<FrCfg>(x00, x10);
            const fe y01 = fe_add<FrCfg>(x01, x11);
            const fe y11 = fe_mul<FrCfg>(fe_sub<FrCfg>(x01, x11), wi);
            sts(p00, fe_add<FrCfg>(y00, y01));
            sts(p01, fe_sub<FrCfg>(y00, y01));
            sts(p10, fe_add<FrCfg>(y10, y11));
            sts(p11, fe_sub<FrCfg>(y10, y11));
        }
        __syncthreads();
        sp = -1;
    }
    if (sp == 0) {  // odd number of stages in this pass: one radix-2 stage on neighbouring elements
        for (uint32_t t = threadIdx.x; t < (uint32_t)(E >> 1); t += blockDim.x) {
            const uint32_t qq = t & Q_mask;
            const uint32_t r = t >> q_log;
            const uint32_t p0 = ((r << 1) << q_log) | qq, p1 = (((r << 1) | 1u) << q_log) | qq;
            const size_t lw = (q_base + qq) & lo_mask;
            const fe x0 = lds(p0), x1 = lds(p1);
            sts(p0, fe_add<FrCfg>(x0, x1));
            if (FINAL) {  // stage 0 of the whole transform: twiddle w^0 = 1
                sts(p1, fe_sub<FrCfg>(x0, x1));
            } else {
                const fe w = fe_load_ro(a.tw + (lw << (a.log_n - a.lo - 1)));
                sts(p1, fe_mul<FrCfg>(fe_sub<FrCfg>(x0, x1), w));
            }
        }
        __syncthreads();
    }

    // ---- scatter: same index for inner passes, bit-reversed index after the last stage ------
    for (uint32_t e = threadIdx.x; e < (uint32_t)E; e += blockDim.x) {
        uint32_t qq, m;
        if (a.lo == 0) { qq = e >> t_log; m = e & T_mask; }
        else           { m = e >> q_log; qq = e & Q_mask; }
        const uint32_t q = q_base + qq;
        const size_t idx = ((size_t)(q >> a.lo) << a.hi) | ((size_t)m << a.lo) | (q & lo_mask);
        const uint32_t pos = (m << q_log) | qq;
        const uint4 u = plane_lo[pos], v = plane_hi[pos];
        fe y;
        y.l[0] = u.x; y.l[1] = u.y; y.l[2] = u.z; y.l[3] = u.w;
        y.l[4] = v.x; y.l[5] = v.y; y.l[6] = v.z; y.l[7] = v.w;
        size_t oi = idx;
        if (FINAL) {
            // bit-reverse over log_n bits (log_n <= 32 handled with 64-bit brev)
            oi = (size_t)(__brevll((unsigned long long)idx) >> (64 - a.log_n));
            if (a.post) y = fe_mul<FrCfg>(y, fe_load_ro(a.post + oi));
            else if (a.has_post_scalar) y = fe_mul<FrCfg>(y, a.post_scalar);
        }
        fe_store(out + oi, y);
    }
}

// Forcing a fourth resident block per SM (64 registers, with spills) was measured slower.
template <bool FINAL>
__global__ void __launch_bounds__(256) ntt_pass_kernel(PassArgs a) {
    extern __shared__ uint4 smem[];
    const TileGeom g = tile_geom(a);
    const int E = g.E;
    uint4* plane_lo = smem;
    uint4* plane_hi = smem + E;
    const uint32_t q_base = blockIdx.x << g.q_log;
    const fe* in = a.in + (size_t)blockIdx.y * a.batch_stride;
    fe* out = a.out + (size_t)blockIdx.y * a.batch_stride;

    // ---- gather the tile -------------------------------------------------------------------
    // a thread's (up to) four elements are all requested before the first one is consumed: one trip to L2 / HBM per
    // tile instead of four dependent ones
    {
        fe v[4];
        uint32_t pos[4];
        size_t gidx[4];
        const uint32_t per = ((uint32_t)E + blockDim.x - 1) / blockDim.x;  // <= 4 (E <= 1024, blockDim = min(E / 2, 256) >= E / 4)
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const uint32_t e = threadIdx.x + (uint32_t)k * blockDim.x;
            if ((uint32_t)k < per && e < (uint32_t)E) {
                tile_slot(a, g, q_base, e, &gidx[k], &pos[k]);
                v[k] = fe_load(in + gidx[k]);
            }
        }
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const uint32_t e = threadIdx.x + (uint32_t)k * blockDim.x;
            if ((uint32_t)k < per && e < (uint32_t)E) {
                fe x = v[k];
                if (a.pre) x = fe_mul<FrCfg>(x, fe_load_ro(a.pre + gidx[k]));
                plane_lo[pos[k]] = make_uint4(x.l[0], x.l[1], x.l[2], x.l[3]);
                plane_hi[pos[k]] = make_uint4(x.l[4], x.l[5], x.l[6], x.l[7]);
            }
        }
    }
    __syncthreads();
    tile_compute<FINAL>(a, g, plane_lo, plane_hi, q_base, out);
}

// A persistent variant of this pass (two blocks per SM walking the tiles, the next tile prefetched with cp.async into the
// other half of a double buffer) was built, passed the parity suite and lost: ~100 registers and twice the shared memory
// leave 2 resident blocks per SM instead of 3, and the pass is bound by the integer-multiply pipe, not by load latency
// (the code is in the history at commit bd42500).

// table[i] = base^i (Montgomery), i < n: thread i multiplies the pow2[b] = base^(2^b) it needs
struct PowArgs {
    fe pow2[32];
    fe scale;  // every entry is multiplied by this (Montgomery one, or n^-1)
};
__global__ void powers_kernel(fe* out, size_t n, PowArgs p) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    fe acc = p.scale;
    for (int b = 0; b < 32; ++b)
        if ((i >> b) & 1) acc = fe_mul<FrCfg>(acc, p.pow2[b]);
    fe_store(out + i, acc);
}

}  // namespace

// ---------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------
fe host_root_of_unity(unsigned log_n) {
    // TWO_ADIC_ROOT_OF_UNITY = 5^((r-1)/2^28) (SURVEY.md §8(a5)); squared down to order 2^log_n
    fe c;
    const uint32_t canon[8] = {0x725b19f0u, 0x9bd61b6eu, 0x41112ed4u, 0x402d111eu,
                               0x8ef62abcu, 0x00e0a7ebu, 0xa58a7e85u, 0x2a3c09f0u};
    for (int i = 0; i < 8; ++i) c.l[i] = canon[i];
    fe w = fe_to_mont<FrCfg>(c);
    for (unsigned i = log_n; i < 28; ++i) w = fe_sqr<FrCfg>(w);
    return w;
}

void fill_powers(fe* d_out, size_t n, fe base, fe scale, cudaStream_t st) {
    PowArgs p;
    p.scale = scale;
    fe b = base;
    for (int i = 0; i < 32; ++i) {
        p.pow2[i] = b;
        b = fe_sqr<FrCfg>(b);
    }
    if (n == 0) return;
    const unsigned bs = 256;
    B200_LAUNCH(powers_kernel, (unsigned)((n + bs - 1) / bs), bs, 0, st)(d_out, n, p);
}

Domain::~Domain() {
    cudaFree(tw_fwd);
    cudaFree(tw_inv);
    cudaFree(coset_fwd);
    cudaFree(coset_inv);
}

int domain_create(unsigned log_n, cudaStream_t st, Domain** out) {
    if (log_n > 28) return B200_ERR_INVALID;
    // every domain is created on its context's device, under that context's lock: the opt-in for the tile's
    // shared memory is (re)applied here, per device, instead of behind a process-wide flag
    if (cudaFuncSetAttribute(ntt_pass_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 32 << kTileLog) != cudaSuccess ||
        cudaFuncSetAttribute(ntt_pass_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 32 << kTileLog) != cudaSuccess)
        return B200_ERR_CUDA;
    Domain* d = new Domain();
    d->log_n = log_n;
    const size_t n = (size_t)1 << log_n;
    const size_t half = n > 1 ? n / 2 : 1;
    if (cudaMalloc(&d->tw_fwd, half * sizeof(fe)) != cudaSuccess ||
        cudaMalloc(&d->tw_inv, half * sizeof(fe)) != cudaSuccess ||
        cudaMalloc(&d->coset_fwd, n * sizeof(fe)) != cudaSuccess ||
        cudaMalloc(&d->coset_inv, n * sizeof(fe)) != cudaSuccess) {
        delete d;
        return B200_ERR_CUDA;
    }
    const fe one = fe_one<FrCfg>();
    const fe w = host_root_of_unity(log_n);
    const fe w_inv = fe_inv<FrCfg>(w);
    fe nn = fe_zero();
    nn.l[0] = (uint32_t)(n & 0xffffffffu);
    nn.l[1] = (uint32_t)(n >> 32);
    d->n_inv = fe_inv<FrCfg>(fe_to_mont<FrCfg>(nn));
    const fe g = fe_from_u32<FrCfg>(5);  // Fr::GENERATOR
    const fe g_inv = fe_inv<FrCfg>(g);
    fill_powers(d->tw_fwd, half, w, one, st);
    fill_powers(d->tw_inv, half, w_inv, one, st);
    fill_powers(d->coset_fwd, n, g, one, st);
    fill_powers(d->coset_inv, n, g_inv, d->n_inv, st);
    d->group_gen = w;
    if (cudaStreamSynchronize(st) != cudaSuccess) {
        delete d;
        return B200_ERR_CUDA;
    }
    *out = d;
    return B200_OK;
}

// CUDA caps gridDim.y at 65535: a larger batch is launched in chunks of at most this many transforms
constexpr unsigned kMaxBatchPerLaunch = 65535;

// the passes of `batch` <= kMaxBatchPerLaunch transforms, one grid row per transform
static int ntt_launch(const Domain* d, fe* data, fe* scratch, int inverse, int coset, unsigned batch, size_t stride,
                      cudaStream_t st) {
    const int L = (int)d->log_n;
    const int P = (L + kTileLog - 1) / kTileLog;
    const int e_log = L < kTileLog ? L : kTileLog;
    const int base = L / P, extra = L % P;
    int hi = L;
    for (int p = 0; p < P; ++p) {
        const int w = base + (p < extra ? 1 : 0);
        PassArgs a;
        a.log_n = L;
        a.hi = hi;
        a.lo = hi - w;
        a.e_log = e_log;
        a.tw = inverse ? d->tw_inv : d->tw_fwd;
        a.pre = (p == 0 && coset && !inverse) ? d->coset_fwd : nullptr;
        a.post = nullptr;
        a.has_post_scalar = 0;
        a.post_scalar = d->n_inv;
        a.batch_stride = stride;
        const bool final_pass = (p == P - 1);
        // inner passes run in place; the pass before the last writes to scratch so that the last
        // (bit-reversing, hence out-of-place) pass lands back in `data`.  A single-pass transform
        // fits one block, which reads its whole tile before writing, so it is in place too.
        a.in = (P > 1 && final_pass) ? scratch : data;
        a.out = (P > 1 && p == P - 2) ? scratch : data;
        if (final_pass && inverse) {
            if (coset) a.post = d->coset_inv;
            else a.has_post_scalar = 1;
        }
        const unsigned E = 1u << e_log;
        unsigned threads = E / 2 < 256 ? E / 2 : 256;
        if (threads < 32) threads = 32;
        dim3 grid((unsigned)(((size_t)1 << L) >> e_log), batch);
        const size_t smem = (size_t)E * 32;
        if (final_pass) {
            B200_LAUNCH(ntt_pass_kernel<true>, grid, threads, smem, st)(a);
        } else {
            B200_LAUNCH(ntt_pass_kernel<false>, grid, threads, smem, st)(a);
        }
        hi -= w;
    }
    return cudaGetLastError() == cudaSuccess ? B200_OK : B200_ERR_CUDA;
}

// data: batch transforms of n elements, `stride` elements apart, transformed in place.
// scratch: at least (batch-1)*stride + n elements when log_n > kTileLog.
int ntt_device(const Domain* d, fe* data, fe* scratch, int inverse, int coset, unsigned batch,
               size_t stride, cudaStream_t st) {
    if (d->log_n == 0 || batch == 0) return B200_OK;  // size-1 transform is the identity (n^-1 = 1)
    for (unsigned first = 0; first < batch; first += kMaxBatchPerLaunch) {
        const unsigned rows = batch - first < kMaxBatchPerLaunch ? batch - first : kMaxBatchPerLaunch;
        const size_t off = (size_t)first * stride;
        const int rc = ntt_launch(d, data + off, scratch + off, inverse, coset, rows, stride, st);
        if (rc != B200_OK) return rc;
    }
    return B200_OK;
}

}  // namespace b200
