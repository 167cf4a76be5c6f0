// C ABI of libb200prover (declared in include/b200prover.h).  Every entry point catches C++
// exceptions, records a thread-local message and returns an error code: nothing unwinds across
// the boundary into the Rust host.
#include <cstring>
#include <new>
#include <string>
#include <vector>

#include "b200prover.h"
#include "device_ctx.h"
#include "transcript.h"

namespace b200 {

static thread_local std::string g_last_error;
std::atomic<uint64_t> g_kernel_launches{0};
std::atomic<uint64_t> g_launch_host_ns{0};
std::atomic<uint64_t> g_graph_launches{0};
std::atomic<uint64_t> g_object_ids{1};
thread_local uint64_t t_kernel_launches = 0;

void set_error(const std::string& msg) { g_last_error = msg; }

int cuda_fail(cudaError_t e, const char* what) {
    g_last_error = std::string(what) + ": " + cudaGetErrorString(e);
    return B200_ERR_CUDA;
}

Context::~Context() {
    for (ProofGraphSet* g : graph_sets) delete g;
    for (auto& kv : domains) delete kv.second;
    if (ntt_ev_init) {
        cudaEventDestroy(ntt_ev[0]);
        cudaEventDestroy(ntt_ev[1]);
    }
    if (ev_fork) cudaEventDestroy(ev_fork);
    if (ev_join) cudaEventDestroy(ev_join);
    if (stream2) cudaStreamDestroy(stream2);
    if (heavy) cudaStreamDestroy(heavy);
    if (hv_fork) cudaEventDestroy(hv_fork);
    if (hv_join) cudaEventDestroy(hv_join);
    if (stream) cudaStreamDestroy(stream);
}

int get_domain(Context* c, unsigned log_n, Domain** out) {
    auto it = c->domains.find(log_n);
    if (it != c->domains.end()) {
        *out = it->second;
        return B200_OK;
    }
    Domain* d = nullptr;
    int rc = domain_create(log_n, c->stream, &d);
    if (rc != B200_OK) {
        if (g_last_error.empty()) set_error("domain_create failed");
        return rc;
    }
    c->domains[log_n] = d;
    *out = d;
    return B200_OK;
}

// ---- field self-test kernels -------------------------------------------------------------------
__device__ __forceinline__ uint64_t st_splitmix(uint64_t seed, uint64_t j) {
    uint64_t z = seed + (j + 1) * 0x9E3779B97F4A7C15ULL;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ULL;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBULL;
    return z ^ (z >> 31);
}
template <class C>
__device__ __forceinline__ fe st_random_fe(uint64_t seed, uint64_t i) {
    fe v;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const uint64_t x = st_splitmix(seed, 4 * i + k);
        v.l[2 * k] = (uint32_t)x;
        v.l[2 * k + 1] = (uint32_t)(x >> 32);
    }
    v.l[7] &= 0x0fffffffu;  // < 2^252 < p: a valid residue without a reduction loop
    return v;
}
__global__ void selftest_field_kernel(uint64_t seed, size_t iters, unsigned long long* mismatches) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= iters) return;
    unsigned long long bad = 0;
    {
        fe a = st_random_fe<FrCfg>(seed, 2 * i), b = st_random_fe<FrCfg>(seed, 2 * i + 1);
        if (i == 0) {  // p - 1 squared: the largest operands
            for (int k = 0; k < 8; ++k) a.l[k] = b.l[k] = FrCfg::mod(k);
            a.l[0] -= 1;
            b.l[0] -= 1;
        }
        if (!fe_eq(fe_mul<FrCfg>(a, b), fe_mul_chain<FrCfg>(a, b))) ++bad;
        if (!fe_eq(fe_sqr<FrCfg>(a), fe_mul_chain<FrCfg>(a, a))) ++bad;  // dedicated squarer
        if (!fe_eq(fe_sqr<FrCfg>(b), fe_mul_chain<FrCfg>(b, b))) ++bad;
    }
    {
        fe a = st_random_fe<FqCfg>(seed ^ 0x5151, 2 * i), b = st_random_fe<FqCfg>(seed ^ 0x5151, 2 * i + 1);
        if (i == 0) {
            for (int k = 0; k < 8; ++k) a.l[k] = b.l[k] = FqCfg::mod(k);
            a.l[0] -= 1;
            b.l[0] -= 1;
        }
        if (!fe_eq(fe_mul<FqCfg>(a, b), fe_mul_chain<FqCfg>(a, b))) ++bad;
        if (!fe_eq(fe_sqr<FqCfg>(a), fe_mul_chain<FqCfg>(a, a))) ++bad;
        if (!fe_eq(fe_sqr<FqCfg>(b), fe_mul_chain<FqCfg>(b, b))) ++bad;
        // fused a*b + c*d / a*b - c*d vs two separate products
        const fe c = st_random_fe<FqCfg>(seed ^ 0x7777, 2 * i), d = i == 0 ? a : st_random_fe<FqCfg>(seed ^ 0x7777, 2 * i + 1);
        if (!fe_eq(fe_mul_add2<FqCfg>(a, b, c, d), fe_add<FqCfg>(fe_mul_chain<FqCfg>(a, b), fe_mul_chain<FqCfg>(c, d)))) ++bad;
        if (!fe_eq(fe_mul_sub2<FqCfg>(a, b, c, d), fe_sub<FqCfg>(fe_mul_chain<FqCfg>(a, b), fe_mul_chain<FqCfg>(c, d)))) ++bad;
    }
    if (bad) atomicAdd(mismatches, bad);
}

// ops 5 and 6 pair element i with element n - 1 - i, so one call reaches the fused two-product forms
template <class C>
__global__ void field_op_kernel(int op, const fe* a, const fe* b, size_t n, fe* out) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const fe x = fe_load(a + i), y = fe_load(b + i);
    fe r;
    switch (op) {
        case 0: r = fe_mul<C>(x, y); break;
        case 1: r = fe_add<C>(x, y); break;
        case 2: r = fe_sub<C>(x, y); break;
        case 3: r = fe_inv<C>(x); break;
        case 4: r = fe_sqr<C>(x); break;
        case 5: r = fe_mul_add2<C>(x, y, fe_load(a + (n - 1 - i)), fe_load(b + (n - 1 - i))); break;
        default: r = fe_mul_sub2<C>(x, y, fe_load(a + (n - 1 - i)), fe_load(b + (n - 1 - i))); break;
    }
    fe_store(out + i, r);
}

}  // namespace b200

using namespace b200;


extern "C" {

const char* b200_last_error(void) { return g_last_error.c_str(); }
const char* b200_version(void) { return "libb200prover 0.1.0 sm_90a"; }

uint64_t b200_kernel_launches(void) { return g_kernel_launches.load(std::memory_order_relaxed); }
uint64_t b200_launch_host_ns(void) { return g_launch_host_ns.load(std::memory_order_relaxed); }
uint64_t b200_graph_launches(void) { return g_graph_launches.load(std::memory_order_relaxed); }
int b200_ctx_use_graphs(b200_ctx* ctx, int on) {
    if (!ctx) return B200_ERR_INVALID;
    std::lock_guard<std::mutex> lk(ctx->c.mu);
    ctx->c.use_graphs = on ? 1 : 0;
    return B200_OK;
}

void b200_keccak256(const uint8_t* data, size_t len, uint8_t out[32]) { Keccak256::hash(data, len, out); }

int b200_init(int device, b200_ctx** out) {
    B200_TRY
    if (!out) return B200_ERR_INVALID;
    int count = 0;
    cudaError_t e = cudaGetDeviceCount(&count);
    if (e != cudaSuccess || count == 0) {
        set_error(std::string("no CUDA device: ") + (e != cudaSuccess ? cudaGetErrorString(e) : "count = 0") +
                  " (libb200prover has no CPU fallback)");
        return B200_ERR_NO_DEVICE;
    }
    if (device < 0 || device >= count) {
        set_error("device ordinal out of range");
        return B200_ERR_INVALID;
    }
    B200_CUDA(cudaSetDevice(device));
    b200_ctx* ctx = new b200_ctx();
    ctx->c.device = device;
    // The context's own stream runs at the highest priority and carries the short, latency-bound kernels
    // (sorts, scans, bucket reduction, transcript-driven glue); the long throughput-bound kernels (bucket
    // accumulation, the side-stream coset NTTs) go to a lowest-priority companion stream.  With several
    // contexts proving on one GPU the block scheduler then slots a proof's short kernels in as soon as
    // SM resources free up instead of queueing them behind another proof's big grid.
    int prio_least = 0, prio_greatest = 0;
    cudaDeviceGetStreamPriorityRange(&prio_least, &prio_greatest);
    const char* pe = std::getenv("B200_STREAM_PRIORITIES");
    const bool prio = !(pe && pe[0] == '0');
    e = cudaStreamCreateWithPriority(&ctx->c.stream, cudaStreamNonBlocking, prio ? prio_greatest : 0);
    if (e == cudaSuccess && prio) {
        e = cudaStreamCreateWithPriority(&ctx->c.heavy, cudaStreamNonBlocking, prio_least);
        if (e == cudaSuccess) e = cudaEventCreateWithFlags(&ctx->c.hv_fork, cudaEventDisableTiming);
        if (e == cudaSuccess) e = cudaEventCreateWithFlags(&ctx->c.hv_join, cudaEventDisableTiming);
    }
    if (e != cudaSuccess) {
        delete ctx;
        return cuda_fail(e, "cudaStreamCreate");
    }
    ctx->c.msm.hv_stream = ctx->c.heavy;
    ctx->c.heavy_plonk = prio && !(pe && pe[0] == '1');  // B200_STREAM_PRIORITIES=1: accumulation only
    ctx->c.msm.hv_fork = ctx->c.hv_fork;
    ctx->c.msm.hv_join = ctx->c.hv_join;
    ctx->c.batch.msm.hv_stream = ctx->c.heavy;
    ctx->c.batch.msm.hv_fork = ctx->c.hv_fork;
    ctx->c.batch.msm.hv_join = ctx->c.hv_join;
    *out = ctx;
    return B200_OK;
    B200_CATCH
}

void b200_shutdown(b200_ctx* ctx) {
    if (!ctx) return;
    cudaSetDevice(ctx->c.device);
    cudaStreamSynchronize(ctx->c.stream);
    delete ctx;
}

// ---- SRS ------------------------------------------------------------------------------------
static bool rd_u32(const uint8_t* b, size_t len, size_t off, uint32_t* v) {
    if (off + 4 > len) return false;
    *v = (uint32_t)b[off] | ((uint32_t)b[off + 1] << 8) | ((uint32_t)b[off + 2] << 16) | ((uint32_t)b[off + 3] << 24);
    return true;
}
static bool rd_u64(const uint8_t* b, size_t len, size_t off, uint64_t* v) {
    uint32_t lo, hi;
    if (!rd_u32(b, len, off, &lo) || !rd_u32(b, len, off + 4, &hi)) return false;
    *v = (uint64_t)lo | ((uint64_t)hi << 32);
    return true;
}

int b200_srs_parse_ptau(const uint8_t* bytes, size_t len, const uint8_t** g1_records, size_t* n_records) {
    B200_TRY
    if (!bytes || !g1_records || !n_records) return B200_ERR_INVALID;
    // header (srs.rs:74-92)
    if (len < 12 || std::memcmp(bytes, "ptau", 4) != 0) {
        set_error("ptau: bad magic");
        return B200_ERR_FORMAT;
    }
    uint32_t version, n_sections;
    rd_u32(bytes, len, 4, &version);
    rd_u32(bytes, len, 8, &n_sections);
    if (version != 1) {
        set_error("Invalid version, cannot parse ptau files of version != 1");
        return B200_ERR_FORMAT;
    }
    if (n_sections != 11) {
        set_error("Invalid number of sections");
        return B200_ERR_FORMAT;
    }
    size_t off = 12;
    // section 1 (srs.rs:95-118)
    uint32_t sec;
    uint64_t size;
    if (!rd_u32(bytes, len, off, &sec) || !rd_u64(bytes, len, off + 4, &size) || sec != 1) {
        set_error("Invalid section number");
        return B200_ERR_FORMAT;
    }
    off += 12;
    uint32_t mod_bytes;
    if (!rd_u32(bytes, len, off, &mod_bytes) || mod_bytes != 32 || off + 4 + 32 + 8 > len) {
        set_error("ptau: bad modulus length");
        return B200_ERR_FORMAT;
    }
    for (int i = 0; i < 8; ++i) {
        uint32_t limb;
        rd_u32(bytes, len, off + 4 + 4 * i, &limb);
        if (limb != FqCfg::mod(i)) {
            set_error("ptau: modulus is not the BN254 base field");
            return B200_ERR_FORMAT;
        }
    }
    uint32_t power;
    rd_u32(bytes, len, off + 4 + 32, &power);
    if (power < 17) {  // MAX_SRS_POWER, srs.rs:44,112
        set_error("ptau: power < 17");
        return B200_ERR_FORMAT;
    }
    if (size > len - off) {  // untrusted 64-bit length: never let `off` wrap or leave the buffer
        set_error("ptau: section 1 longer than the file");
        return B200_ERR_FORMAT;
    }
    off += (size_t)size;
    // section 2 (srs.rs:124-141)
    if (!rd_u32(bytes, len, off, &sec) || !rd_u64(bytes, len, off + 4, &size) || sec != 2) {
        set_error("Invalid section number");
        return B200_ERR_FORMAT;
    }
    off += 12;
    size_t avail = len > off ? len - off : 0;
    if (avail > size) avail = size;
    *g1_records = bytes + off;
    *n_records = avail / 64;
    return B200_OK;
    B200_CATCH
}

int b200_bases_load(b200_ctx* ctx, const uint8_t* points64, size_t n, int window_bits, int check_on_curve,
                    b200_bases** out) {
    B200_TRY
    if (!ctx || !points64 || !out) return B200_ERR_INVALID;
    if (window_bits != 0 && window_bits != 1 && (window_bits < 8 || window_bits > 23)) {
        set_error("window_bits must be 0 (auto, throughput), 1 (auto, latency) or in [8, 23]");
        return B200_ERR_INVALID;
    }
    std::lock_guard<std::mutex> lk(ctx->c.mu);
    B200_CUDA(cudaSetDevice(ctx->c.device));
    Bases* b = nullptr;
    int rc = bases_create(reinterpret_cast<const g1_affine*>(points64), n, window_bits, check_on_curve,
                          ctx->c.stream, &b);
    if (rc != B200_OK) return rc;
    *out = new b200_bases{b};
    return B200_OK;
    B200_CATCH
}

int b200_bases_load_device(b200_ctx* ctx, const void* d_points64, size_t n, int window_bits, b200_bases** out) {
    B200_TRY
    if (!ctx || !d_points64 || !out) return B200_ERR_INVALID;
    if (window_bits != 0 && window_bits != 1 && (window_bits < 8 || window_bits > 23)) {
        set_error("window_bits must be 0 (auto, throughput), 1 (auto, latency) or in [8, 23]");
        return B200_ERR_INVALID;
    }
    std::lock_guard<std::mutex> lk(ctx->c.mu);
    B200_CUDA(cudaSetDevice(ctx->c.device));
    Bases* b = nullptr;
    int rc = bases_create_device(reinterpret_cast<const g1_affine*>(d_points64), n, window_bits, ctx->c.stream, &b);
    if (rc != B200_OK) return rc;
    *out = new b200_bases{b};
    return B200_OK;
    B200_CATCH
}

void b200_bases_free(b200_ctx* ctx, b200_bases* bases) {
    if (!bases) return;
    if (ctx) {
        std::lock_guard<std::mutex> lk(ctx->c.mu);
        cudaSetDevice(ctx->c.device);
        cudaStreamSynchronize(ctx->c.stream);
        delete bases->b;
    } else {
        delete bases->b;
    }
    delete bases;
}

size_t b200_bases_len(const b200_bases* bases) { return bases ? bases->b->n : 0; }

void b200_bases_plan(const b200_bases* bases, int plan[4]) {
    if (!bases || !plan) return;
    plan[0] = bases->b->plan.c;
    plan[1] = bases->b->plan.n_digits;
    plan[2] = bases->b->plan.n_phys;
    plan[3] = bases->b->plan.n_tables;
}

// ---- MSM ------------------------------------------------------------------------------------
static void store_point(const g1_affine& p, uint64_t out_xy[8]) { std::memcpy(out_xy, &p, 64); }

int b200_msm_device(b200_ctx* ctx, const b200_bases* bases, size_t base_off, const void* d_scalars, size_t n,
                    int scalars_montgomery, uint64_t out_xy[8], int* out_is_identity) {
    B200_TRY
    if (!ctx || !bases || !out_xy || (n && !d_scalars)) return B200_ERR_INVALID;
    std::lock_guard<std::mutex> lk(ctx->c.mu);
    B200_CUDA(cudaSetDevice(ctx->c.device));
    g1_affine r;
    int inf = 0;
    int rc = msm_device(bases->b, base_off, reinterpret_cast<const fe*>(d_scalars), n, scalars_montgomery,
                        &ctx->c.msm, ctx->c.stream, &r, &inf);
    if (rc != B200_OK) return rc;
    store_point(r, out_xy);
    if (out_is_identity) *out_is_identity = inf;
    return B200_OK;
    B200_CATCH
}

int b200_msm(b200_ctx* ctx, const b200_bases* bases, size_t base_off, const uint64_t* scalars, size_t n,
             int scalars_montgomery, uint64_t out_xy[8], int* out_is_identity) {
    B200_TRY
    if (!ctx || !bases || !out_xy || (n && !scalars)) return B200_ERR_INVALID;
    std::lock_guard<std::mutex> lk(ctx->c.mu);
    B200_CUDA(cudaSetDevice(ctx->c.device));
    int rc = ctx->c.msm.scalars.reserve(n * sizeof(fe) + 32);
    if (rc != B200_OK) return rc;
    if (n) B200_CUDA(cudaMemcpyAsync(ctx->c.msm.scalars.p, scalars, n * sizeof(fe), cudaMemcpyHostToDevice, ctx->c.stream));
    g1_affine r;
    int inf = 0;
    rc = msm_device(bases->b, base_off, reinterpret_cast<const fe*>(ctx->c.msm.scalars.p), n, scalars_montgomery,
                    &ctx->c.msm, ctx->c.stream, &r, &inf);
    if (rc != B200_OK) return rc;
    store_point(r, out_xy);
    if (out_is_identity) *out_is_identity = inf;
    return B200_OK;
    B200_CATCH
}

int b200_g1_sum_affine(const uint64_t* points_xy, const int* is_identity, size_t k, uint64_t out_xy[8],
                       int* out_is_identity) {
    B200_TRY
    if ((k && !points_xy) || !out_xy) return B200_ERR_INVALID;
    g1_xyzz acc = g1_xyzz_inf();
    for (size_t i = 0; i < k; ++i) {
        if (is_identity && is_identity[i]) continue;
        g1_affine p;
        std::memcpy(&p, points_xy + 8 * i, 64);
        acc = g1_add_mixed(acc, p);
    }
    const g1_affine r = g1_to_affine(acc);
    store_point(r, out_xy);
    if (out_is_identity) *out_is_identity = g1_xyzz_is_inf(acc) ? 1 : 0;
    return B200_OK;
    B200_CATCH
}

int b200_msm_batch_device(b200_ctx* ctx, const b200_bases* bases, size_t base_off, const void* d_scalars, size_t n,
                          size_t stride, unsigned batch, int scalars_montgomery, uint64_t* out_xy,
                          int* out_is_identity) {
    B200_TRY
    if (!ctx || !bases || !out_xy || (n && !d_scalars) || batch == 0 || batch > 64 || stride < n) return B200_ERR_INVALID;
    std::lock_guard<std::mutex> lk(ctx->c.mu);
    B200_CUDA(cudaSetDevice(ctx->c.device));
    std::vector<g1_affine> r(batch);
    std::vector<int> inf(batch, 0);
    int rc = msm_device_batch(bases->b, base_off, reinterpret_cast<const fe*>(d_scalars), n, stride, batch,
                              scalars_montgomery, &ctx->c.msm, ctx->c.stream, r.data(), inf.data());
    if (rc != B200_OK) return rc;
    std::memcpy(out_xy, r.data(), (size_t)batch * 64);
    if (out_is_identity)
        for (unsigned i = 0; i < batch; ++i) out_is_identity[i] = inf[i];
    return B200_OK;
    B200_CATCH
}

int b200_msm_timing_totals(b200_ctx* ctx, int reset, double out[3]) {
    B200_TRY
    if (!ctx) return B200_ERR_INVALID;
    std::lock_guard<std::mutex> lk(ctx->c.mu);
    // the single calls' scratch and the batch calls' (b200_plonk_prove_batch, b200_plonk_link_batch)
    MsmScratch* const scratches[2] = {&ctx->c.msm, &ctx->c.batch.msm};
    if (out) {
        out[0] = out[1] = out[2] = 0;
        for (const MsmScratch* s : scratches) {
            out[0] += s->tot_acc_ms;
            out[1] += s->tot_pairs;
            out[2] += s->tot_launches;
        }
    }
    if (reset)
        for (MsmScratch* s : scratches) s->tot_acc_ms = s->tot_pairs = s->tot_launches = 0;
    return B200_OK;
    B200_CATCH
}

int b200_msm_tuning(b200_ctx* ctx, int throughput_mode) {
    B200_TRY
    if (!ctx) return B200_ERR_INVALID;
    // kept for ABI compatibility: the tree reduction (msm.cu) has one setting for lone MSMs and the prover alike
    (void)throughput_mode;
    return B200_OK;
    B200_CATCH
}

int b200_msm_timing(b200_ctx* ctx, int enable, float out_ms[4]) {
    B200_TRY
    if (!ctx) return B200_ERR_INVALID;
    std::lock_guard<std::mutex> lk(ctx->c.mu);
    ctx->c.msm.timing = enable != 0;
    ctx->c.batch.msm.timing = enable != 0;  // the batch calls commit through their own scratch
    if (out_ms)
        for (int i = 0; i < 4; ++i) out_ms[i] = ctx->c.msm.ms[i];
    return B200_OK;
    B200_CATCH
}

// ---- NTT ------------------------------------------------------------------------------------
// caller holds ctx->c.mu
static int ntt_device_locked(b200_ctx* ctx, void* d_data, unsigned log_n, int inverse, int coset, unsigned batch,
                             size_t stride) {
    const size_t n = (size_t)1 << log_n;
    B200_CUDA(cudaSetDevice(ctx->c.device));
    Domain* d = nullptr;
    int rc = get_domain(&ctx->c, log_n, &d);
    if (rc != B200_OK) return rc;
    rc = ctx->c.ntt_scratch.reserve(((size_t)(batch - 1) * stride + n) * sizeof(fe));
    if (rc != B200_OK) return rc;
    if (!ctx->c.ntt_ev_init) {
        B200_CUDA(cudaEventCreate(&ctx->c.ntt_ev[0]));
        B200_CUDA(cudaEventCreate(&ctx->c.ntt_ev[1]));
        ctx->c.ntt_ev_init = true;
    }
    cudaEventRecord(ctx->c.ntt_ev[0], ctx->c.stream);
    rc = ntt_device(d, reinterpret_cast<fe*>(d_data), reinterpret_cast<fe*>(ctx->c.ntt_scratch.p), inverse, coset,
                    batch, stride, ctx->c.stream);
    cudaEventRecord(ctx->c.ntt_ev[1], ctx->c.stream);
    if (rc != B200_OK) {
        set_error("ntt kernel launch failed");
        return rc;
    }
    B200_CUDA(cudaStreamSynchronize(ctx->c.stream));
    cudaEventElapsedTime(&ctx->c.ntt_last_ms, ctx->c.ntt_ev[0], ctx->c.ntt_ev[1]);
    return B200_OK;
}

int b200_ntt_device(b200_ctx* ctx, void* d_data, unsigned log_n, int inverse, int coset, unsigned batch,
                    size_t stride) {
    B200_TRY
    if (!ctx || !d_data || log_n > 28 || batch == 0) return B200_ERR_INVALID;
    if (stride < ((size_t)1 << log_n)) {
        set_error("ntt: stride < n");
        return B200_ERR_INVALID;
    }
    std::lock_guard<std::mutex> lk(ctx->c.mu);
    return ntt_device_locked(ctx, d_data, log_n, inverse, coset, batch, stride);
    B200_CATCH
}

int b200_ntt(b200_ctx* ctx, uint64_t* data, unsigned log_n, int inverse, int coset) {
    B200_TRY
    if (!ctx || !data || log_n > 28) return B200_ERR_INVALID;
    const size_t n = (size_t)1 << log_n;
    // one critical section: upload, transform and download cannot interleave with another caller's
    // (whose reserve() could otherwise free the staging buffer under this call)
    std::lock_guard<std::mutex> lk(ctx->c.mu);
    B200_CUDA(cudaSetDevice(ctx->c.device));
    int rc = ctx->c.ntt_data.reserve(n * sizeof(fe));
    if (rc != B200_OK) return rc;
    B200_CUDA(cudaMemcpyAsync(ctx->c.ntt_data.p, data, n * sizeof(fe), cudaMemcpyHostToDevice, ctx->c.stream));
    rc = ntt_device_locked(ctx, ctx->c.ntt_data.p, log_n, inverse, coset, 1, n);
    if (rc != B200_OK) return rc;
    B200_CUDA(cudaMemcpyAsync(data, ctx->c.ntt_data.p, n * sizeof(fe), cudaMemcpyDeviceToHost, ctx->c.stream));
    B200_CUDA(cudaStreamSynchronize(ctx->c.stream));
    return B200_OK;
    B200_CATCH
}

int b200_ntt_last_ms(b200_ctx* ctx, float* out_ms) {
    if (!ctx || !out_ms) return B200_ERR_INVALID;
    *out_ms = ctx->c.ntt_last_ms;
    return B200_OK;
}

int b200_domain_generator(b200_ctx* ctx, unsigned log_n, uint64_t out[4]) {
    B200_TRY
    if (!ctx || !out || log_n > 28) return B200_ERR_INVALID;
    std::lock_guard<std::mutex> lk(ctx->c.mu);
    B200_CUDA(cudaSetDevice(ctx->c.device));
    Domain* d = nullptr;
    int rc = get_domain(&ctx->c, log_n, &d);
    if (rc != B200_OK) return rc;
    std::memcpy(out, &d->group_gen, 32);
    return B200_OK;
    B200_CATCH
}

// ---- synthetic inputs -------------------------------------------------------------------------
int b200_splitmix_fr_device(b200_ctx* ctx, uint64_t seed, size_t first, size_t n, int montgomery, void* d_out) {
    B200_TRY
    if (!ctx || (n && !d_out)) return B200_ERR_INVALID;
    std::lock_guard<std::mutex> lk(ctx->c.mu);
    B200_CUDA(cudaSetDevice(ctx->c.device));
    int rc = splitmix_fr_device(seed, first, n, montgomery, reinterpret_cast<fe*>(d_out), ctx->c.stream);
    if (rc != B200_OK) return rc;
    B200_CUDA(cudaStreamSynchronize(ctx->c.stream));
    return B200_OK;
    B200_CATCH
}

int b200_known_dlog_bases_device(b200_ctx* ctx, uint64_t seed, size_t first, size_t n, void* d_out) {
    B200_TRY
    if (!ctx || (n && !d_out)) return B200_ERR_INVALID;
    std::lock_guard<std::mutex> lk(ctx->c.mu);
    B200_CUDA(cudaSetDevice(ctx->c.device));
    int rc = g1_known_dlog_bases_device(seed, first, n, reinterpret_cast<g1_affine*>(d_out), ctx->c.stream);
    if (rc != B200_OK) return rc;
    B200_CUDA(cudaStreamSynchronize(ctx->c.stream));
    return B200_OK;
    B200_CATCH
}

// ---- self-test ----------------------------------------------------------------------------------
int b200_selftest_field(b200_ctx* ctx, uint64_t seed, size_t iters, uint64_t* mismatches) {
    B200_TRY
    if (!ctx || !mismatches) return B200_ERR_INVALID;
    std::lock_guard<std::mutex> lk(ctx->c.mu);
    B200_CUDA(cudaSetDevice(ctx->c.device));
    unsigned long long* d_bad = nullptr;
    B200_CUDA(cudaMalloc(&d_bad, 8));
    cudaMemsetAsync(d_bad, 0, 8, ctx->c.stream);
    if (iters) B200_LAUNCH(selftest_field_kernel, (unsigned)((iters + 127) / 128), 128, 0, ctx->c.stream)(seed, iters, d_bad);
    unsigned long long h = 0;
    cudaMemcpyAsync(&h, d_bad, 8, cudaMemcpyDeviceToHost, ctx->c.stream);
    cudaError_t e = cudaStreamSynchronize(ctx->c.stream);
    cudaFree(d_bad);
    if (e != cudaSuccess) return cuda_fail(e, "selftest_field");
    *mismatches = h;
    return B200_OK;
    B200_CATCH
}

int b200_field_op(b200_ctx* ctx, int field, int op, const uint64_t* a, const uint64_t* b, size_t n, uint64_t* out) {
    B200_TRY
    if (!ctx || !a || !b || !out || field < 0 || field > 1 || op < 0 || op > 6) return B200_ERR_INVALID;
    if (n == 0) return B200_OK;
    std::lock_guard<std::mutex> lk(ctx->c.mu);
    B200_CUDA(cudaSetDevice(ctx->c.device));
    fe *da = nullptr, *db = nullptr, *dout = nullptr;
    B200_CUDA(cudaMalloc(&da, n * sizeof(fe)));
    B200_CUDA(cudaMalloc(&db, n * sizeof(fe)));
    B200_CUDA(cudaMalloc(&dout, n * sizeof(fe)));
    cudaMemcpyAsync(da, a, n * sizeof(fe), cudaMemcpyHostToDevice, ctx->c.stream);
    cudaMemcpyAsync(db, b, n * sizeof(fe), cudaMemcpyHostToDevice, ctx->c.stream);
    const unsigned bs = 128, grid = (unsigned)((n + bs - 1) / bs);
    if (field == 0) B200_LAUNCH(field_op_kernel<FrCfg>, grid, bs, 0, ctx->c.stream)(op, da, db, n, dout);
    else B200_LAUNCH(field_op_kernel<FqCfg>, grid, bs, 0, ctx->c.stream)(op, da, db, n, dout);
    cudaMemcpyAsync(out, dout, n * sizeof(fe), cudaMemcpyDeviceToHost, ctx->c.stream);
    cudaError_t e = cudaStreamSynchronize(ctx->c.stream);
    cudaFree(da);
    cudaFree(db);
    cudaFree(dout);
    if (e != cudaSuccess) return cuda_fail(e, "field_op");
    return B200_OK;
    B200_CATCH
}

}  // extern "C"
