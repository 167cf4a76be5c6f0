// Batch Poseidon2 hashing over the BN254 scalar field (SURVEY.md §8(f) f4: the witness-side hashing
// that dominates once MSM/NTT are on the device).
//
// Replaces, for batches of independent hashes, the reference's native
//   crypto::hash::Poseidon2Sponge::{hash, absorb, squeeze, permute}
//     /root/reference/crates/crypto/src/hash/poseidon2.rs:25-209
//   crypto::hash::compute_poseidon_hash        /root/reference/crates/crypto/src/hash/mod.rs:12-18
// with t = 3 (RATE 2, CAPACITY 1), R_F = 8, R_P = 56, alpha = 5 (constants.rs:15-36).  One thread
// per hash: a permutation is 80 S-boxes = 240 Fr products plus additions, integer-pipe bound like
// everything else here; constants live in __constant__ memory.
#include <cstring>

#include "b200prover.h"
#include <mutex>

#include "device_ctx.h"
#include "poseidon2_constants.h"

namespace b200 {

namespace {

__constant__ uint32_t c_full_rc[24][8];
__constant__ uint32_t c_partial_rc[56][8];

using Fr = FrCfg;

__device__ __forceinline__ fe rc_full(int i) {
    fe r;
#pragma unroll
    for (int k = 0; k < 8; ++k) r.l[k] = c_full_rc[i][k];
    return r;
}
__device__ __forceinline__ fe rc_partial(int i) {
    fe r;
#pragma unroll
    for (int k = 0; k < 8; ++k) r.l[k] = c_partial_rc[i][k];
    return r;
}
__device__ __forceinline__ fe sbox(const fe& x) {  // x^5 (poseidon2.rs:201-208)
    const fe x2 = fe_sqr<Fr>(x);
    return fe_mul<Fr>(fe_sqr<Fr>(x2), x);
}
// M_E = circ(2,1,1): add the sum of the state to every element (poseidon2.rs:146-152)
__device__ __forceinline__ void external_mds(fe s[3]) {
    const fe sum = fe_add<Fr>(fe_add<Fr>(s[0], s[1]), s[2]);
#pragma unroll
    for (int i = 0; i < 3; ++i) s[i] = fe_add<Fr>(s[i], sum);
}
// M_I = [[2,1,1],[1,2,1],[1,1,3]] (poseidon2.rs:187-195)
__device__ __forceinline__ void internal_mds(fe s[3]) {
    const fe sum = fe_add<Fr>(fe_add<Fr>(s[0], s[1]), s[2]);
    s[2] = fe_dbl<Fr>(s[2]);
#pragma unroll
    for (int i = 0; i < 3; ++i) s[i] = fe_add<Fr>(s[i], sum);
}
// poseidon2.rs:90-110
__device__ void permute(fe s[3]) {
    external_mds(s);
    for (int r = 0; r < 4; ++r) {
#pragma unroll
        for (int i = 0; i < 3; ++i) s[i] = sbox(fe_add<Fr>(s[i], rc_full(3 * r + i)));
        external_mds(s);
    }
    for (int r = 0; r < 56; ++r) {
        s[0] = sbox(fe_add<Fr>(s[0], rc_partial(r)));
        internal_mds(s);
    }
    for (int r = 4; r < 8; ++r) {
#pragma unroll
        for (int i = 0; i < 3; ++i) s[i] = sbox(fe_add<Fr>(s[i], rc_full(3 * r + i)));
        external_mds(s);
    }
}

__global__ void __launch_bounds__(128) k_poseidon2_permute(fe* states, size_t batch) {
    const size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= batch) return;
    fe s[3];
    for (int i = 0; i < 3; ++i) s[i] = fe_load(states + 3 * t + i);
    permute(s);
    for (int i = 0; i < 3; ++i) fe_store(states + 3 * t + i, s[i]);
}

// Poseidon2Sponge::hash: absorb `len` scalars at rate 2 (permuting when the rate is full), then one
// squeeze = permute and return state[CAPACITY] (poseidon2.rs:38-84)
__global__ void __launch_bounds__(128) k_poseidon2_hash(const fe* __restrict__ in, size_t batch, size_t len,
                                                        fe* __restrict__ out) {
    const size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= batch) return;
    fe s[3] = {fe_zero(), fe_zero(), fe_zero()};
    int next = 0;
    const fe* x = in + t * len;
    for (size_t i = 0; i < len; ++i) {
        if (next == 2) {
            permute(s);
            next = 0;
        }
        s[next + 1] = fe_add<Fr>(s[next + 1], fe_load_ro(x + i));
        ++next;
    }
    permute(s);
    fe_store(out + t, s[1]);
}

// two-to-one sponge hash H(a, b): absorb two scalars at rate 2, squeeze one (one permutation)
__device__ __forceinline__ fe hash2(const fe& a, const fe& b) {
    fe s[3] = {fe_zero(), a, b};
    permute(s);
    return s[1];
}

// Merkle roots of `batch` openings (circuit-types `MerkleOpening<HEIGHT>`; native side of
// circuits-core/src/zk_gadgets/primitives/merkle.rs:13-126): cur = leaf hash; per level the sister node and whether
// the running hash is the RIGHT child:  cur = H(sister, cur)  or  H(cur, sister).
__global__ void __launch_bounds__(128) k_merkle_roots(const fe* __restrict__ leaf_hashes, const fe* __restrict__ sisters,
                                                      const uint8_t* __restrict__ is_right, size_t batch, unsigned height,
                                                      fe* __restrict__ roots) {
    const size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= batch) return;
    fe cur = fe_load_ro(leaf_hashes + t);
    for (unsigned lvl = 0; lvl < height; ++lvl) {
        const fe sis = fe_load_ro(sisters + t * height + lvl);
        cur = is_right[t * height + lvl] ? hash2(sis, cur) : hash2(cur, sis);
    }
    fe_store(roots + t, cur);
}

// `count` consecutive values of `batch` Poseidon CSPRNG streams (darkpool-types/src/csprng.rs:30-75): value i of a
// stream is H(seed, i); out[s * count + j] = H(seed_s, first_index_s + j).  Indices are small integers (u64).
__global__ void __launch_bounds__(128) k_csprng(const fe* __restrict__ seeds, const uint64_t* __restrict__ first_index,
                                                size_t batch, size_t count, fe* __restrict__ out) {
    const size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= batch * count) return;
    const size_t sidx = t / count, j = t % count;
    const uint64_t idx = first_index[sidx] + j;
    fe i_canon = fe_zero();
    i_canon.l[0] = (uint32_t)idx;
    i_canon.l[1] = (uint32_t)(idx >> 32);
    fe_store(out + t, hash2(fe_load_ro(seeds + sidx), fe_to_mont<Fr>(i_canon)));
}

// one upload per device, whatever context gets there first; a failed upload leaves the flag clear and the next call
// on that device tries again
std::mutex g_constants_mu[64];
bool g_constants_loaded[64];  // guarded by g_constants_mu[device]

}  // namespace

// The upload runs on the caller's stream and is waited for before the device is marked loaded: a pageable
// cudaMemcpyToSymbol on the legacy stream may return before its DMA lands, and the legacy stream does not order the
// non-blocking context streams the kernels run on (this one's, or another context's that waited on the lock).
static int upload_constants(cudaStream_t st) {
    B200_CUDA(cudaMemcpyToSymbolAsync(c_full_rc, kPoseidon2FullRc, sizeof(kPoseidon2FullRc), 0, cudaMemcpyHostToDevice, st));
    B200_CUDA(cudaMemcpyToSymbolAsync(c_partial_rc, kPoseidon2PartialRc, sizeof(kPoseidon2PartialRc), 0,
                                      cudaMemcpyHostToDevice, st));
    B200_CUDA(cudaStreamSynchronize(st));
    return B200_OK;
}
static int load_constants(int device, cudaStream_t st) {
    if (device < 0 || device >= 64) return upload_constants(st);
    std::lock_guard<std::mutex> lk(g_constants_mu[device]);  // the context mutex does not cover other contexts
    if (g_constants_loaded[device]) return B200_OK;
    const int rc = upload_constants(st);
    if (rc == B200_OK) g_constants_loaded[device] = true;
    return rc;
}

}  // namespace b200

using namespace b200;

extern "C" {

int b200_poseidon2_permute_batch(b200_ctx* ctx, uint64_t* states, size_t batch) {
    B200_TRY
    if (!ctx || (batch && !states)) return B200_ERR_INVALID;
    if (batch == 0) return B200_OK;
    std::lock_guard<std::mutex> lk(ctx->c.mu);
    B200_ENTER(ctx->c);
    cudaStream_t st = ctx->c.stream;
    int rc = load_constants(ctx->c.device, st);
    if (rc != B200_OK) return rc;
    if ((rc = ctx->c.plonk_ws.reserve(batch * 3 * sizeof(fe))) != B200_OK) return rc;
    fe* d = reinterpret_cast<fe*>(ctx->c.plonk_ws.p);
    B200_CUDA(cudaMemcpyAsync(d, states, batch * 3 * sizeof(fe), cudaMemcpyDefault, st));
    B200_LAUNCH(k_poseidon2_permute, (unsigned)((batch + 127) / 128), 128, 0, st)(d, batch);
    B200_CUDA(cudaMemcpyAsync(states, d, batch * 3 * sizeof(fe), cudaMemcpyDefault, st));
    B200_CUDA(cudaStreamSynchronize(st));
    return B200_OK;
    B200_CATCH
}

int b200_poseidon2_hash_batch(b200_ctx* ctx, const uint64_t* inputs, size_t batch, size_t len, uint64_t* out) {
    B200_TRY
    if (!ctx || !out || (batch && len && !inputs)) return B200_ERR_INVALID;
    if (batch == 0) return B200_OK;
    std::lock_guard<std::mutex> lk(ctx->c.mu);
    B200_ENTER(ctx->c);
    cudaStream_t st = ctx->c.stream;
    int rc = load_constants(ctx->c.device, st);
    if (rc != B200_OK) return rc;
    if ((rc = ctx->c.plonk_ws.reserve((batch * len + batch + 1) * sizeof(fe))) != B200_OK) return rc;
    fe* d_in = reinterpret_cast<fe*>(ctx->c.plonk_ws.p);
    fe* d_out = d_in + batch * len;
    if (len) B200_CUDA(cudaMemcpyAsync(d_in, inputs, batch * len * sizeof(fe), cudaMemcpyDefault, st));
    B200_LAUNCH(k_poseidon2_hash, (unsigned)((batch + 127) / 128), 128, 0, st)(d_in, batch, len, d_out);
    B200_CUDA(cudaMemcpyAsync(out, d_out, batch * sizeof(fe), cudaMemcpyDefault, st));
    B200_CUDA(cudaStreamSynchronize(st));
    return B200_OK;
    B200_CATCH
}

int b200_poseidon2_merkle_root_batch(b200_ctx* ctx, const uint64_t* leaf_hashes, const uint64_t* sisters,
                                     const uint8_t* is_right, size_t batch, unsigned height, uint64_t* roots) {
    B200_TRY
    if (!ctx || !roots || (batch && (!leaf_hashes || (height && (!sisters || !is_right)))) || height > 64) return B200_ERR_INVALID;
    if (batch == 0) return B200_OK;
    std::lock_guard<std::mutex> lk(ctx->c.mu);
    B200_ENTER(ctx->c);
    cudaStream_t st = ctx->c.stream;
    int rc = load_constants(ctx->c.device, st);
    if (rc != B200_OK) return rc;
    const size_t n_sis = batch * height;
    if ((rc = ctx->c.plonk_ws.reserve((2 * batch + n_sis + 1) * sizeof(fe) + n_sis + 64)) != B200_OK) return rc;
    fe* d_leaf = reinterpret_cast<fe*>(ctx->c.plonk_ws.p);
    fe* d_sis = d_leaf + batch;
    fe* d_out = d_sis + n_sis;
    uint8_t* d_bits = reinterpret_cast<uint8_t*>(d_out + batch);
    B200_CUDA(cudaMemcpyAsync(d_leaf, leaf_hashes, batch * sizeof(fe), cudaMemcpyDefault, st));
    if (n_sis) {
        B200_CUDA(cudaMemcpyAsync(d_sis, sisters, n_sis * sizeof(fe), cudaMemcpyDefault, st));
        B200_CUDA(cudaMemcpyAsync(d_bits, is_right, n_sis, cudaMemcpyDefault, st));
    }
    B200_LAUNCH(k_merkle_roots, (unsigned)((batch + 127) / 128), 128, 0, st)(d_leaf, d_sis, d_bits, batch, height, d_out);
    B200_CUDA(cudaMemcpyAsync(roots, d_out, batch * sizeof(fe), cudaMemcpyDefault, st));
    B200_CUDA(cudaStreamSynchronize(st));
    return B200_OK;
    B200_CATCH
}

int b200_poseidon2_csprng_batch(b200_ctx* ctx, const uint64_t* seeds, const uint64_t* first_index, size_t batch, size_t count,
                                uint64_t* out) {
    B200_TRY
    if (!ctx || !out || (batch && (!seeds || !first_index))) return B200_ERR_INVALID;
    if (batch == 0 || count == 0) return B200_OK;
    std::lock_guard<std::mutex> lk(ctx->c.mu);
    B200_ENTER(ctx->c);
    cudaStream_t st = ctx->c.stream;
    int rc = load_constants(ctx->c.device, st);
    if (rc != B200_OK) return rc;
    const size_t total = batch * count;
    if ((rc = ctx->c.plonk_ws.reserve((batch + total + 1) * sizeof(fe) + batch * 8 + 64)) != B200_OK) return rc;
    fe* d_seeds = reinterpret_cast<fe*>(ctx->c.plonk_ws.p);
    fe* d_out = d_seeds + batch;
    uint64_t* d_idx = reinterpret_cast<uint64_t*>(d_out + total);
    B200_CUDA(cudaMemcpyAsync(d_seeds, seeds, batch * sizeof(fe), cudaMemcpyDefault, st));
    B200_CUDA(cudaMemcpyAsync(d_idx, first_index, batch * 8, cudaMemcpyDefault, st));
    B200_LAUNCH(k_csprng, (unsigned)((total + 127) / 128), 128, 0, st)(d_seeds, d_idx, batch, count, d_out);
    B200_CUDA(cudaMemcpyAsync(out, d_out, total * sizeof(fe), cudaMemcpyDefault, st));
    B200_CUDA(cudaStreamSynchronize(st));
    return B200_OK;
    B200_CATCH
}

}  // extern "C"
