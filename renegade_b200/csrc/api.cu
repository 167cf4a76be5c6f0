// C ABI of libb200prover (declared in include/b200prover.h).  Every entry point catches C++
// exceptions, records a thread-local message and returns an error code: nothing unwinds across
// the boundary into the Rust host.
#include <cudaTypedefs.h>

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
thread_local const std::atomic<bool>* t_cancel = nullptr;

void set_error(const std::string& msg) { g_last_error = msg; }

int cancelled(Context* c) {
    for (cudaStream_t s : {c->stream, c->stream2, c->heavy})
        if (s) cudaStreamSynchronize(s);
    set_error("cancelled (B200_ERR_CANCELLED): the job was cancelled before it finished");
    return B200_ERR_CANCELLED;
}

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

int b200_init(int device, b200_ctx** out) { return b200::context_create(device, /*express=*/false, nullptr, out); }

}  // extern "C"

// ---- SM partitions ----------------------------------------------------------------------------------
// The green-context calls of the driver API are looked up through the runtime (cudaGetDriverEntryPointByVersion) rather
// than linked from libcuda: the library then loads, and refuses arguments, on a machine without a driver, and takes the
// driver the runtime has already loaded.
namespace {
struct Driver {
    PFN_cuDeviceGet_v2000 device_get = nullptr;
    PFN_cuCtxGetCurrent_v4000 ctx_get_current = nullptr;
    PFN_cuCtxSetCurrent_v4000 ctx_set_current = nullptr;
    PFN_cuGetErrorString_v6000 error_string = nullptr;
    PFN_cuDeviceGetDevResource_v12040 device_get_resource = nullptr;
    PFN_cuDevSmResourceSplitByCount_v12040 sm_split_by_count = nullptr;
    PFN_cuDevResourceGenerateDesc_v12040 generate_desc = nullptr;
    PFN_cuGreenCtxCreate_v12040 green_create = nullptr;
    PFN_cuGreenCtxDestroy_v12040 green_destroy = nullptr;
    PFN_cuCtxFromGreenCtx_v12040 ctx_from_green = nullptr;
    PFN_cuGreenCtxGetDevResource_v12040 green_get_resource = nullptr;
    PFN_cuGreenCtxStreamCreate_v12050 green_stream_create = nullptr;
    std::string missing;  // the first entry point the driver did not give; empty when all are there
};

template <class F>
void lookup(Driver& d, const char* name, unsigned version, F* f) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q = cudaDriverEntryPointSymbolNotFound;
    if (cudaGetDriverEntryPointByVersion(name, &p, version, cudaEnableDefault, &q) != cudaSuccess ||
        q != cudaDriverEntryPointSuccess || !p) {
        cudaGetLastError();
        if (d.missing.empty()) d.missing = name;
        return;
    }
    *f = reinterpret_cast<F>(p);
}

const Driver& driver() {
    static const Driver d = [] {
        Driver x;
        lookup(x, "cuDeviceGet", 2000, &x.device_get);
        lookup(x, "cuCtxGetCurrent", 4000, &x.ctx_get_current);
        lookup(x, "cuCtxSetCurrent", 4000, &x.ctx_set_current);
        lookup(x, "cuGetErrorString", 6000, &x.error_string);
        lookup(x, "cuDeviceGetDevResource", 12040, &x.device_get_resource);
        lookup(x, "cuDevSmResourceSplitByCount", 12040, &x.sm_split_by_count);
        lookup(x, "cuDevResourceGenerateDesc", 12040, &x.generate_desc);
        lookup(x, "cuGreenCtxCreate", 12040, &x.green_create);
        lookup(x, "cuGreenCtxDestroy", 12040, &x.green_destroy);
        lookup(x, "cuCtxFromGreenCtx", 12040, &x.ctx_from_green);
        lookup(x, "cuGreenCtxGetDevResource", 12040, &x.green_get_resource);
        lookup(x, "cuGreenCtxStreamCreate", 12050, &x.green_stream_create);
        return x;
    }();
    return d;
}

int driver_ready(const char* who) {
    const Driver& d = driver();
    if (d.missing.empty()) return B200_OK;
    set_error(std::string(who) + ": the CUDA driver has no " + d.missing + " (green contexts need CUDA 12.5 or later)");
    return B200_ERR_CUDA;
}

int cu_fail(CUresult r, const char* what) {
    const char* s = nullptr;
    if (driver().error_string) driver().error_string(r, &s);
    set_error(std::string(what) + ": " + (s ? s : "CUresult " + std::to_string((int)r)));
    return B200_ERR_CUDA;
}

// cudaGetDeviceCount and the ordinal's range, with the messages of b200_init
int check_device(int device) {
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
    return B200_OK;
}

// A context's teardown: its streams, events and buffers inside its partition, then the green context itself
void context_destroy(b200_ctx* ctx) {
    CUgreenCtx g = ctx->c.green;
    {
        Enter in(ctx->c);
        cudaStreamSynchronize(ctx->c.stream);
        delete ctx;
    }
    if (g) driver().green_destroy(g);
}

// One block's SM into a 256-bit mask; every block then holds its SM a few microseconds so that the grid spreads over
// every SM the launch may use
__global__ void probe_sms_kernel(unsigned long long* mask) {
    if (threadIdx.x == 0) {
        unsigned smid;
        asm volatile("mov.u32 %0, %%smid;" : "=r"(smid));
        atomicOr(mask + ((smid >> 6) & 3), 1ull << (smid & 63));
    }
    const long long t0 = clock64();
    while (clock64() - t0 < 20000) {
    }
}
}  // namespace

b200::Enter::Enter(const Context& c) {
    if (!c.green) {
        const cudaError_t e = cudaSetDevice(c.device);
        if (e != cudaSuccess) rc = cuda_fail(e, "cudaSetDevice");
        return;
    }
    const Driver& d = driver();  // complete: the context was made through it
    if (d.ctx_get_current(&prev) != CUDA_SUCCESS) prev = nullptr;
    const CUresult r = d.ctx_set_current(c.green_cu);
    if (r != CUDA_SUCCESS) {
        rc = cu_fail(r, "cuCtxSetCurrent(green context)");
        return;
    }
    restore = true;
}

b200::Enter::~Enter() {
    if (restore) driver().ctx_set_current(prev);
}

int b200::stream_create(const Context& c, int prio, cudaStream_t* out) {
    if (!c.green) B200_CUDA(cudaStreamCreateWithPriority(out, cudaStreamNonBlocking, prio));
    else {
        CUstream s = nullptr;
        const CUresult r = driver().green_stream_create(&s, c.green, CU_STREAM_NON_BLOCKING, prio);
        if (r != CUDA_SUCCESS) return cu_fail(r, "cuGreenCtxStreamCreate");
        *out = s;
    }
    return B200_OK;
}

int b200::sm_split(int device, unsigned first_sms, SmGroup groups[2]) {
    int rc = check_device(device);
    if (rc != B200_OK || (rc = driver_ready("sm_split")) != B200_OK) return rc;
    B200_CUDA(cudaSetDevice(device));  // the primary context, which the green contexts retain, is up before them
    B200_CUDA(cudaFree(nullptr));
    const Driver& d = driver();
    CUdevice dev = 0;
    CUresult r = d.device_get(&dev, device);
    CUdevResource all{}, split[2]{};
    if (r == CUDA_SUCCESS) r = d.device_get_resource(dev, &all, CU_DEV_RESOURCE_TYPE_SM);
    if (r != CUDA_SUCCESS) return cu_fail(r, "cuDeviceGetDevResource");
    if (first_sms + 8 > all.sm.smCount) {
        set_error("express_sms must leave at least 8 SMs for the normal group: the device has " + std::to_string(all.sm.smCount));
        return B200_ERR_INVALID;
    }
    unsigned n_groups = 1;
    r = d.sm_split_by_count(&split[0], &n_groups, &all, &split[1], 0, first_sms);
    if (r != CUDA_SUCCESS || n_groups != 1) return cu_fail(r, "cuDevSmResourceSplitByCount");
    if (split[1].sm.smCount < 8) {
        set_error("express_sms must leave at least 8 SMs for the normal group: the split of " + std::to_string(all.sm.smCount) +
                  " SMs gave " + std::to_string(split[0].sm.smCount) + " and " + std::to_string(split[1].sm.smCount));
        return B200_ERR_INVALID;
    }
    for (int i = 0; i < 2; ++i) {
        if ((r = d.generate_desc(&groups[i].desc, &split[i], 1)) != CUDA_SUCCESS) return cu_fail(r, "cuDevResourceGenerateDesc");
        groups[i].sms = split[i].sm.smCount;
    }
    return B200_OK;
}

int b200::probe_sms(Context* c, uint64_t mask[4]) {
    B200_ENTER(*c);
    int sms = (int)c->sms;
    if (!sms) B200_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, c->device));
    unsigned long long* d_mask = nullptr;
    B200_CUDA(cudaMalloc(&d_mask, 32));
    cudaError_t e = cudaMemsetAsync(d_mask, 0, 32, c->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(c->stream);
    const cudaStream_t streams[3] = {c->stream, c->heavy, c->stream2};
    for (cudaStream_t st : streams) {
        if (!st || e != cudaSuccess) continue;
        B200_LAUNCH(probe_sms_kernel, 8 * (unsigned)sms, 128, 0, st)(d_mask);  // eagerly
        cudaGraph_t g = nullptr;
        cudaGraphExec_t x = nullptr;
        e = cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal);
        if (e == cudaSuccess) {
            B200_LAUNCH(probe_sms_kernel, 8 * (unsigned)sms, 128, 0, st)(d_mask);  // captured, then replayed
            e = cudaStreamEndCapture(st, &g);
        }
        if (e == cudaSuccess) e = cudaGraphInstantiate(&x, g, 0);
        if (e == cudaSuccess) {
            e = cudaGraphLaunch(x, st);
            g_graph_launches.fetch_add(1, std::memory_order_relaxed);
        }
        if (e == cudaSuccess) e = cudaStreamSynchronize(st);
        if (x) cudaGraphExecDestroy(x);
        if (g) cudaGraphDestroy(g);
    }
    unsigned long long h[4] = {};
    if (e == cudaSuccess) e = cudaMemcpy(h, d_mask, 32, cudaMemcpyDeviceToHost);
    cudaFree(d_mask);
    if (e != cudaSuccess) return cuda_fail(e, "probe_sms");
    for (int i = 0; i < 4; ++i) mask[i] |= h[i];
    return B200_OK;
}

int b200::context_create(int device, bool express, const SmGroup* group, b200_ctx** out) {
    B200_TRY
    if (!out) return B200_ERR_INVALID;
    int rc = check_device(device);
    if (rc != B200_OK) return rc;
    B200_CUDA(cudaSetDevice(device));
    b200_ctx* ctx = new b200_ctx();
    ctx->c.device = device;
    if (group) {
        const Driver& d = driver();
        CUdevice dev = 0;
        CUdevResource res{};
        CUresult r = d.device_get(&dev, device);
        if (r == CUDA_SUCCESS) r = d.green_create(&ctx->c.green, group->desc, dev, CU_GREEN_CTX_DEFAULT_STREAM);
        if (r == CUDA_SUCCESS) r = d.ctx_from_green(&ctx->c.green_cu, ctx->c.green);
        if (r == CUDA_SUCCESS) r = d.green_get_resource(ctx->c.green, &res, CU_DEV_RESOURCE_TYPE_SM);
        if (r != CUDA_SUCCESS) {
            rc = cu_fail(r, "green context");
            context_destroy(ctx);
            return rc;
        }
        ctx->c.sms = res.sm.smCount;
    }
    Enter in(ctx->c);
    if (in.rc != B200_OK) {
        context_destroy(ctx);
        return in.rc;
    }
    // The context's own stream runs at the highest priority and carries the short, latency-bound kernels
    // (sorts, scans, bucket reduction, transcript-driven glue); the long throughput-bound kernels (bucket
    // accumulation, the side-stream coset NTTs) go to a lowest-priority companion stream.  With several
    // contexts proving on one GPU the block scheduler then slots a proof's short kernels in as soon as
    // SM resources free up instead of queueing them behind another proof's big grid.
    // An express context (a pool's express worker) ranks each stream role above a normal context's where the device has
    // the levels: the companion one level above the least priority, and with priorities off its one stream at the
    // greatest instead of 0.  The main stream is at the greatest for both.  Lower numbers are higher priorities.
    int prio_least = 0, prio_greatest = 0;
    cudaDeviceGetStreamPriorityRange(&prio_least, &prio_greatest);
    const char* pe = std::getenv("B200_STREAM_PRIORITIES");
    const bool prio = !(pe && pe[0] == '0');
    const bool lift = express && prio_least - prio_greatest >= 1;  // at least two levels
    const int main_prio = prio ? prio_greatest : (lift ? prio_greatest : 0);
    const int heavy_prio = lift ? prio_least - 1 : prio_least;
    ctx->c.stream2_prio = prio ? heavy_prio : main_prio;
    rc = stream_create(ctx->c, main_prio, &ctx->c.stream);
    if (rc == B200_OK && prio) {
        rc = stream_create(ctx->c, heavy_prio, &ctx->c.heavy);
        cudaError_t e = cudaSuccess;
        if (rc == B200_OK) e = cudaEventCreateWithFlags(&ctx->c.hv_fork, cudaEventDisableTiming);
        if (e == cudaSuccess) e = cudaEventCreateWithFlags(&ctx->c.hv_join, cudaEventDisableTiming);
        if (e != cudaSuccess) rc = cuda_fail(e, "cudaEventCreate");
    }
    if (rc != B200_OK) {
        context_destroy(ctx);
        return rc;
    }
    ctx->c.msm.hv_stream = ctx->c.heavy;
    ctx->c.heavy_plonk = prio && !(pe && pe[0] == '1');  // B200_STREAM_PRIORITIES=1: accumulation only
    ctx->c.msm.hv_fork = ctx->c.hv_fork;
    ctx->c.msm.hv_join = ctx->c.hv_join;
    ctx->c.batch.msm.hv_stream = ctx->c.heavy;
    ctx->c.batch.msm.hv_fork = ctx->c.hv_fork;
    ctx->c.batch.msm.hv_join = ctx->c.hv_join;
    ctx->c.msm.sms = ctx->c.batch.msm.sms = ctx->c.sms;
    *out = ctx;
    return B200_OK;
    B200_CATCH
}

extern "C" {

void b200_shutdown(b200_ctx* ctx) {
    if (ctx) context_destroy(ctx);
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

int b200_srs_parse_ptau_g2(const uint8_t* bytes, size_t len, uint64_t g2_h[16], uint64_t g2_tau_h[16]) {
    B200_TRY
    if (!bytes || !g2_h || !g2_tau_h) return B200_ERR_INVALID;
    // header, section 1 and section 2's header: the checks of b200_srs_parse_ptau, which leaves g1 just past the latter
    const uint8_t* g1 = nullptr;
    size_t n_records = 0;
    int rc = b200_srs_parse_ptau(bytes, len, &g1, &n_records);
    if (rc != B200_OK) return rc;
    size_t off = (size_t)(g1 - bytes);
    uint64_t size;
    rd_u64(bytes, len, off - 8, &size);
    if (size > len - off) {  // untrusted 64-bit length, as for section 1
        set_error("ptau: section 2 longer than the file");
        return B200_ERR_FORMAT;
    }
    off += (size_t)size;
    // section 3 (srs.rs:147-157): its header, then h and beta_h
    uint32_t sec;
    if (!rd_u32(bytes, len, off, &sec) || !rd_u64(bytes, len, off + 4, &size)) {
        set_error("ptau: the file ends before section 3");
        return B200_ERR_FORMAT;
    }
    if (sec != 3) {
        set_error("Invalid section number");
        return B200_ERR_FORMAT;
    }
    off += 12;
    if (size < 256) {
        set_error("ptau: section 3 is shorter than its two G2 records");
        return B200_ERR_FORMAT;
    }
    if (len - off < 256) {
        set_error("ptau: the file ends inside section 3's two G2 records");
        return B200_ERR_FORMAT;
    }
    std::memcpy(g2_h, bytes + off, 128);
    std::memcpy(g2_tau_h, bytes + off + 128, 128);
    if (!g2_record_on_curve(g2_h) || !g2_record_on_curve(g2_tau_h)) {
        set_error("ptau: section 3: G2 point not on curve");
        return B200_ERR_NOT_ON_CURVE;
    }
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
    B200_ENTER(ctx->c);
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
    B200_ENTER(ctx->c);
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
        Enter in(ctx->c);
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
    B200_ENTER(ctx->c);
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
    B200_ENTER(ctx->c);
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
    B200_ENTER(ctx->c);
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
    B200_ENTER(ctx->c);
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
    B200_ENTER(ctx->c);
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
    B200_ENTER(ctx->c);
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
    B200_ENTER(ctx->c);
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
    B200_ENTER(ctx->c);
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
    B200_ENTER(ctx->c);
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
    B200_ENTER(ctx->c);
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
