// Copy-constraint permutation from a circuit's wiring, on the device (b200_plonk_preprocess_wiring).
//
// A finalized circuit names the variable on every wire position p = i*n + j (wire i, row j).  The positions of one
// variable, in ascending p, form one cycle of the permutation: each maps to the next, the last to the first.  The
// positions are grouped by a stable sort of the 64-bit keys (variable << 32 | position) — a radix sort, so the result
// does not depend on scheduling — and one kernel links each group into its cycle.
#include <cub/device/device_radix_sort.cuh>

#include "device_ctx.h"

namespace b200 {

namespace {

constexpr uint32_t kNoBadIndex = 0xFFFFFFFFu;

// keys[p] = var << 32 | p; *bad = the lowest position whose variable index is out of range (kNoBadIndex: none)
__global__ void k_wiring_keys(const uint32_t* __restrict__ wire_vars, uint32_t count, uint32_t num_vars,
                              uint64_t* __restrict__ keys, uint32_t* __restrict__ bad) {
    const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= count) return;
    const uint32_t v = __ldg(wire_vars + p);
    if (v >= num_vars) atomicMin(bad, p);
    keys[p] = (uint64_t)v << 32 | p;
}

// sorted keys -> perm[pos] = the next position of the same variable, the group's first position for its last
__global__ void k_wiring_cycles(const uint64_t* __restrict__ keys, uint32_t count, uint64_t* __restrict__ perm) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= count) return;
    const uint64_t key = __ldg(keys + t);
    const uint32_t var = (uint32_t)(key >> 32);
    uint32_t next;
    if (t + 1 < count && (uint32_t)(__ldg(keys + t + 1) >> 32) == var) {
        next = (uint32_t)__ldg(keys + t + 1);
    } else {
        // first key of the group: the lowest index whose key is >= var << 32
        const uint64_t first = (uint64_t)var << 32;
        uint32_t lo = 0, hi = t;
        while (lo < hi) {
            const uint32_t mid = lo + (hi - lo) / 2;
            if (__ldg(keys + mid) < first) lo = mid + 1;
            else hi = mid;
        }
        next = (uint32_t)__ldg(keys + lo);
    }
    perm[(uint32_t)key] = next;
}

}  // namespace

int wiring_permutation(const uint32_t* d_wire_vars, size_t count, size_t num_vars, uint64_t* d_perm, cudaStream_t st) {
    if (count == 0 || count >= kNoBadIndex || num_vars == 0 || num_vars > kNoBadIndex) {
        set_error("preprocess_wiring: num_vars must be in [1, 2^32) and the wiring at most 2^32 - 2 positions");
        return B200_ERR_INVALID;
    }
    int end_bit = 33;  // the position, and as many bits of the variable index as num_vars - 1 has
    while (end_bit < 64 && ((uint64_t)(num_vars - 1) >> (end_bit - 32))) ++end_bit;
    uint64_t* keys = nullptr;  // count keys in, count keys out, the bad-index word, then the sort's scratch
    size_t temp_bytes = 0;
    cub::DeviceRadixSort::SortKeys(nullptr, temp_bytes, keys, keys, (uint32_t)count, 0, end_bit, st);
    const size_t head = (2 * count + 1) * sizeof(uint64_t);
    cudaError_t e = cudaMalloc(&keys, head + temp_bytes);
    if (e != cudaSuccess) return cuda_fail(e, "cudaMalloc(wiring keys)");
    uint32_t* d_bad = reinterpret_cast<uint32_t*>(keys + 2 * count);
    uint32_t bad = kNoBadIndex;
    const unsigned grid = (unsigned)((count + 255) / 256);
    e = cudaMemcpyAsync(d_bad, &bad, sizeof(bad), cudaMemcpyHostToDevice, st);
    if (e == cudaSuccess) {
        B200_LAUNCH(k_wiring_keys, grid, 256, 0, st)(d_wire_vars, (uint32_t)count, (uint32_t)num_vars, keys, d_bad);
        e = cub::DeviceRadixSort::SortKeys(reinterpret_cast<char*>(keys) + head, temp_bytes, keys, keys + count, (uint32_t)count, 0,
                                           end_bit, st);
    }
    if (e == cudaSuccess) {
        B200_LAUNCH(k_wiring_cycles, grid, 256, 0, st)(keys + count, (uint32_t)count, d_perm);
        e = cudaMemcpyAsync(&bad, d_bad, sizeof(bad), cudaMemcpyDeviceToHost, st);
    }
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    cudaFree(keys);
    if (e != cudaSuccess) return cuda_fail(e, "wiring_permutation");
    if (bad != kNoBadIndex) {
        set_error("preprocess_wiring: wire_vars[" + std::to_string(bad) + "] is not below num_vars = " + std::to_string(num_vars));
        return B200_ERR_INVALID;
    }
    return B200_OK;
}

}  // namespace b200
