// Multi-GPU layer of libb200prover: one MSM sharded by point range over the GPUs of a box, behind the C ABI.
//
// SURVEY.md §8(e): the MSM is a sum over disjoint index ranges of independent terms, so rank g of W owns the
// points [g n / W, (g + 1) n / W) (resident window tables) and receives the matching scalar slice; every GPU
// runs the whole Pippenger locally and contributes ONE group element (128-byte XYZZ record).  Elliptic-curve
// addition is not an NCCL reduction operator, so the exchange is `ncclAllGather` of the W records followed by
// a W-term addition on every device, in rank order — associativity makes the affine result bit-identical to
// the single-GPU MSM (north_star: "a single NCCL reduce of the per-GPU partial sums over NVLink").
//
// Two ways to span the box, one implementation:
//   * b200_multi_init       — ONE host process drives all listed devices (the Rust relayer's shape: boundary
//                             B1 of SURVEY.md §8(b), `b200_init(const int* devs, int n_dev, ...)`); NCCL
//                             communicators from ncclCommInitAll; collectives grouped with ncclGroupStart/End;
//   * b200_multi_init_rank  — one process per GPU (torchrun, bench.py); the 128-byte NCCL unique id is made
//                             by rank 0 (b200_nccl_unique_id) and handed to the others by the host.
// NCCL is bound at run time (dlopen of libnccl.so.2): a process that already holds a copy — PyTorch ships its
// own — shares it instead of mapping a second one, and the single-GPU entry points need no NCCL at all.
#include <dlfcn.h>
#include <nccl.h>

#include <cstring>
#include <memory>
#include <vector>

#include "b200prover.h"
#include "device_ctx.h"

namespace b200 {

namespace {

struct NcclApi {
    void* handle = nullptr;
    ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
    ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
    ncclResult_t (*CommInitAll)(ncclComm_t*, int, const int*) = nullptr;
    ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
    ncclResult_t (*AllGather)(const void*, void*, size_t, ncclDataType_t, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*GroupStart)() = nullptr;
    ncclResult_t (*GroupEnd)() = nullptr;
    const char* (*GetErrorString)(ncclResult_t) = nullptr;
    ncclResult_t (*GetVersion)(int*) = nullptr;
};

std::mutex g_nccl_mu;
NcclApi g_nccl;

int nccl_load() {
    std::lock_guard<std::mutex> lk(g_nccl_mu);
    if (g_nccl.handle) return B200_OK;
    void* h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
    if (!h) h = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
    if (!h) {
        set_error(std::string("NCCL not found: ") + dlerror());
        return B200_ERR_INVALID;
    }
    NcclApi a;
    a.handle = h;
#define B200_NCCL_SYM(field, name)                                    \
    a.field = reinterpret_cast<decltype(a.field)>(dlsym(h, name));    \
    if (!a.field) {                                                   \
        set_error(std::string("NCCL symbol missing: ") + name);       \
        return B200_ERR_INVALID;                                      \
    }
    B200_NCCL_SYM(GetUniqueId, "ncclGetUniqueId")
    B200_NCCL_SYM(CommInitRank, "ncclCommInitRank")
    B200_NCCL_SYM(CommInitAll, "ncclCommInitAll")
    B200_NCCL_SYM(CommDestroy, "ncclCommDestroy")
    B200_NCCL_SYM(AllGather, "ncclAllGather")
    B200_NCCL_SYM(GroupStart, "ncclGroupStart")
    B200_NCCL_SYM(GroupEnd, "ncclGroupEnd")
    B200_NCCL_SYM(GetErrorString, "ncclGetErrorString")
    B200_NCCL_SYM(GetVersion, "ncclGetVersion")
#undef B200_NCCL_SYM
    g_nccl = a;
    return B200_OK;
}

int nccl_fail(ncclResult_t r, const char* what) {
    set_error(std::string(what) + ": " + (g_nccl.GetErrorString ? g_nccl.GetErrorString(r) : "nccl error"));
    return B200_ERR_CUDA;
}
#define B200_NCCL(expr)                                               \
    do {                                                              \
        ncclResult_t _r = (expr);                                     \
        if (_r != ncclSuccess) return nccl_fail(_r, #expr);           \
    } while (0)

// total[0] = sum over ranks of gathered[r], in rank order (every rank computes the same value)
__global__ void k_sum_partials(const g1_xyzz* __restrict__ gathered, int world, g1_xyzz* __restrict__ total) {
    if (threadIdx.x || blockIdx.x) return;
    g1_xyzz acc = g1_xyzz_load(gathered);
    for (int r = 1; r < world; ++r) acc = g1_add(acc, g1_xyzz_load(gathered + r));
    g1_xyzz_store(total, acc);
}

}  // namespace

struct MultiLocal {
    b200_ctx* ctx = nullptr;
    ncclComm_t comm = nullptr;
    int rank = 0;
    DevBuf scalars;   // this rank's scalar slice, when the caller's is in host memory
    DevBuf partial;   // this rank's 128-byte record
    DevBuf gathered;  // world records + the total behind them
    HostPinned h_total;
    cudaEvent_t done = nullptr;
};

}  // namespace b200

using namespace b200;

struct b200_multi {
    int world = 0;
    std::vector<MultiLocal> locals;  // devices driven by this process
    std::mutex mu;
};

struct b200_multi_bases {
    size_t n = 0;  // points of the whole MSM
    std::vector<b200_bases*> shard;   // one per local device
    std::vector<size_t> begin, end;   // its [begin, end) range
};

static void shard_range(size_t n, int rank, int world, size_t* begin, size_t* end) {
    const size_t base = n / (size_t)world, rem = n % (size_t)world;
    *begin = (size_t)rank * base + ((size_t)rank < rem ? (size_t)rank : rem);
    *end = *begin + base + ((size_t)rank < rem ? 1 : 0);
}

static int multi_alloc_local(MultiLocal* l, int world) {
    int rc;
    B200_CUDA(cudaSetDevice(l->ctx->c.device));
    if ((rc = l->partial.reserve(sizeof(g1_xyzz))) != B200_OK) return rc;
    if ((rc = l->gathered.reserve((size_t)(world + 1) * sizeof(g1_xyzz))) != B200_OK) return rc;
    if ((rc = l->h_total.reserve(sizeof(g1_xyzz))) != B200_OK) return rc;
    B200_CUDA(cudaEventCreateWithFlags(&l->done, cudaEventDisableTiming));
    return B200_OK;
}

// The shards of n points over this process's devices, each non-empty one made by load(ctx, begin, count, &shard); every
// shard made so far is freed when one fails.
template <class Load>
static int multi_bases_make(b200_multi* m, size_t n, b200_multi_bases** out, Load&& load) {
    std::lock_guard<std::mutex> lk(m->mu);
    std::unique_ptr<b200_multi_bases> b(new b200_multi_bases());
    b->n = n;
    const size_t nl = m->locals.size();
    b->shard.assign(nl, nullptr);
    b->begin.resize(nl);
    b->end.resize(nl);
    for (size_t i = 0; i < nl; ++i) {
        shard_range(n, m->locals[i].rank, m->world, &b->begin[i], &b->end[i]);
        const size_t cnt = b->end[i] - b->begin[i];
        if (cnt == 0) continue;  // more ranks than points: this shard is empty
        const int rc = load(m->locals[i].ctx, b->begin[i], cnt, &b->shard[i]);
        if (rc != B200_OK) {
            b200_multi_bases_free(m, b.release());
            return rc;
        }
    }
    *out = b.release();
    return B200_OK;
}

extern "C" {

void b200_shard_range(size_t n, int rank, int world, size_t* begin, size_t* end) {
    if (!begin || !end || world <= 0 || rank < 0 || rank >= world) return;
    shard_range(n, rank, world, begin, end);
}

int b200_nccl_version(int* version) {
    B200_TRY
    if (!version) return B200_ERR_INVALID;
    int rc = nccl_load();
    if (rc != B200_OK) return rc;
    B200_NCCL(g_nccl.GetVersion(version));
    return B200_OK;
    B200_CATCH
}

int b200_nccl_unique_id(uint8_t out[128]) {
    B200_TRY
    if (!out) return B200_ERR_INVALID;
    int rc = nccl_load();
    if (rc != B200_OK) return rc;
    static_assert(sizeof(ncclUniqueId) == 128, "NCCL unique id is 128 bytes");
    ncclUniqueId id;
    B200_NCCL(g_nccl.GetUniqueId(&id));
    std::memcpy(out, &id, 128);
    return B200_OK;
    B200_CATCH
}

void b200_multi_shutdown(b200_multi* m) {
    if (!m) return;
    for (MultiLocal& l : m->locals) {
        if (l.ctx) {
            cudaSetDevice(l.ctx->c.device);
            cudaStreamSynchronize(l.ctx->c.stream);
        }
        if (l.comm && g_nccl.CommDestroy) g_nccl.CommDestroy(l.comm);
        if (l.done) cudaEventDestroy(l.done);
        if (l.ctx) b200_shutdown(l.ctx);
    }
    delete m;  // the per-device buffers go with it (cudaFree / cudaFreeHost take pointers of any device)
}

int b200_multi_init(const int* devices, int n_dev, b200_multi** out) {
    B200_TRY
    if (!devices || n_dev <= 0 || n_dev > 64 || !out) {
        set_error("multi_init: need 1..64 device ordinals");
        return B200_ERR_INVALID;
    }
    int rc = nccl_load();
    if (rc != B200_OK) return rc;
    std::unique_ptr<b200_multi> m(new b200_multi());
    m->world = n_dev;
    m->locals.resize(n_dev);
    auto fail = [&](int code) {
        b200_multi_shutdown(m.release());
        return code;
    };
    for (int i = 0; i < n_dev; ++i) {
        m->locals[i].rank = i;
        if ((rc = b200_init(devices[i], &m->locals[i].ctx)) != B200_OK) return fail(rc);
    }
    std::vector<ncclComm_t> comms(n_dev);
    ncclResult_t r = g_nccl.CommInitAll(comms.data(), n_dev, devices);
    if (r != ncclSuccess) return fail(nccl_fail(r, "ncclCommInitAll"));
    for (int i = 0; i < n_dev; ++i) m->locals[i].comm = comms[i];
    for (int i = 0; i < n_dev; ++i)
        if ((rc = multi_alloc_local(&m->locals[i], n_dev)) != B200_OK) return fail(rc);
    *out = m.release();
    return B200_OK;
    B200_CATCH
}

int b200_multi_init_rank(int device, int rank, int world, const uint8_t unique_id[128], b200_multi** out) {
    B200_TRY
    if (!unique_id || !out || world <= 0 || rank < 0 || rank >= world) {
        set_error("multi_init_rank: bad rank / world / id");
        return B200_ERR_INVALID;
    }
    int rc = nccl_load();
    if (rc != B200_OK) return rc;
    std::unique_ptr<b200_multi> m(new b200_multi());
    m->world = world;
    m->locals.resize(1);
    MultiLocal& l = m->locals[0];
    l.rank = rank;
    auto fail = [&](int code) {
        b200_multi_shutdown(m.release());
        return code;
    };
    if ((rc = b200_init(device, &l.ctx)) != B200_OK) return fail(rc);
    ncclUniqueId id;
    std::memcpy(&id, unique_id, 128);
    cudaSetDevice(device);
    ncclResult_t r = g_nccl.CommInitRank(&l.comm, world, id, rank);
    if (r != ncclSuccess) return fail(nccl_fail(r, "ncclCommInitRank"));
    if ((rc = multi_alloc_local(&l, world)) != B200_OK) return fail(rc);
    *out = m.release();
    return B200_OK;
    B200_CATCH
}

int b200_multi_world(const b200_multi* m) { return m ? m->world : 0; }
int b200_multi_local_devices(const b200_multi* m) { return m ? (int)m->locals.size() : 0; }
b200_ctx* b200_multi_ctx(b200_multi* m, int local) {
    if (!m || local < 0 || local >= (int)m->locals.size()) return nullptr;
    return m->locals[local].ctx;
}
int b200_multi_rank(const b200_multi* m, int local) {
    if (!m || local < 0 || local >= (int)m->locals.size()) return -1;
    return m->locals[local].rank;
}

void b200_multi_bases_free(b200_multi* m, b200_multi_bases* b) {
    if (!b) return;
    for (size_t i = 0; i < b->shard.size(); ++i)
        if (b->shard[i]) b200_bases_free(m && i < m->locals.size() ? m->locals[i].ctx : nullptr, b->shard[i]);
    delete b;
}

int b200_multi_bases_load(b200_multi* m, const uint8_t* points64, size_t n, int window_bits, int check_on_curve,
                          b200_multi_bases** out) {
    B200_TRY
    if (!m || !points64 || !out || n == 0) return B200_ERR_INVALID;
    return multi_bases_make(m, n, out, [&](b200_ctx* ctx, size_t begin, size_t cnt, b200_bases** shard) {
        return b200_bases_load(ctx, points64 + 64 * begin, cnt, window_bits, check_on_curve, shard);
    });
    B200_CATCH
}

int b200_multi_bases_known_dlog(b200_multi* m, uint64_t seed, size_t n, int window_bits, b200_multi_bases** out) {
    B200_TRY
    if (!m || !out || n == 0) return B200_ERR_INVALID;
    return multi_bases_make(m, n, out, [&](b200_ctx* ctx, size_t begin, size_t cnt, b200_bases** shard) -> int {
        B200_ENTER(ctx->c);
        void* d_pts = nullptr;
        B200_CUDA(cudaMalloc(&d_pts, cnt * 64));
        int rc = b200_known_dlog_bases_device(ctx, seed, begin, cnt, d_pts);
        if (rc == B200_OK) rc = b200_bases_load_device(ctx, d_pts, cnt, window_bits, shard);
        cudaFree(d_pts);
        return rc;
    });
    B200_CATCH
}

int b200_multi_bases_plan(const b200_multi_bases* b, int local, int plan[4]) {
    if (!b || local < 0 || local >= (int)b->shard.size() || !plan) return B200_ERR_INVALID;
    plan[0] = plan[1] = plan[2] = plan[3] = 0;
    if (b->shard[local]) b200_bases_plan(b->shard[local], plan);
    return B200_OK;
}
size_t b200_multi_bases_len(const b200_multi_bases* b) { return b ? b->n : 0; }
int b200_multi_bases_shard(const b200_multi_bases* b, int local, size_t* begin, size_t* end) {
    if (!b || local < 0 || local >= (int)b->shard.size() || !begin || !end) return B200_ERR_INVALID;
    *begin = b->begin[local];
    *end = b->end[local];
    return B200_OK;
}

// scalars_local[i]: this process's slice for local device i — host pointers (scalars_on_device = 0, copied
// here) or device pointers on that device (1).
static int multi_msm(b200_multi* m, const b200_multi_bases* b, const void* const* scalars_local, int scalars_on_device,
                     int montgomery, uint64_t out_xy[8], int* out_inf) {
    const size_t nl = m->locals.size();
    int rc;
    // the local contexts are used directly: hold their locks (always taken in index order) for the whole call
    std::vector<std::unique_lock<std::mutex>> ctx_locks;
    for (size_t i = 0; i < nl; ++i) ctx_locks.emplace_back(m->locals[i].ctx->c.mu);
    // 1. every local device: (copy its scalar slice,) run its Pippenger — enqueue only, no host wait
    for (size_t i = 0; i < nl; ++i) {
        MultiLocal& l = m->locals[i];
        Context& c = l.ctx->c;
        const size_t cnt = b->end[i] - b->begin[i];
        B200_CUDA(cudaSetDevice(c.device));
        const fe* d_scalars = reinterpret_cast<const fe*>(scalars_local[i]);
        if (cnt && !scalars_on_device) {
            if ((rc = l.scalars.reserve(cnt * sizeof(fe) + 32)) != B200_OK) return rc;
            B200_CUDA(cudaMemcpyAsync(l.scalars.p, scalars_local[i], cnt * sizeof(fe), cudaMemcpyHostToDevice, c.stream));
            d_scalars = reinterpret_cast<const fe*>(l.scalars.p);
        }
        g1_xyzz* partial = reinterpret_cast<g1_xyzz*>(l.partial.p);
        MsmPending launched;  // nothing for msm_finish_batch: the point stays on the device
        rc = cnt ? msm_launch_batch(b->shard[i]->b, 0, d_scalars, cnt, cnt, 1, montgomery, MsmEpilogue::DevicePoint, &c.msm, c.stream,
                                    &launched, partial)
                 : msm_identity_point(partial, c.stream);  // an empty shard contributes the identity
        if (rc != B200_OK) return rc;
    }
    // 2. the exchange: all_gather of the 128-byte records (grouped when this process drives several devices)
    if (m->world > 1) {
        B200_NCCL(g_nccl.GroupStart());
        for (size_t i = 0; i < nl; ++i) {
            MultiLocal& l = m->locals[i];
            ncclResult_t r = g_nccl.AllGather(l.partial.p, l.gathered.p, sizeof(g1_xyzz), ncclUint8, l.comm, l.ctx->c.stream);
            if (r != ncclSuccess) {
                g_nccl.GroupEnd();
                return nccl_fail(r, "ncclAllGather");
            }
        }
        B200_NCCL(g_nccl.GroupEnd());
    }
    // 3. every device adds the W records in rank order; local device 0's total goes to the host
    for (size_t i = 0; i < nl; ++i) {
        MultiLocal& l = m->locals[i];
        Context& c = l.ctx->c;
        B200_CUDA(cudaSetDevice(c.device));
        g1_xyzz* gathered = reinterpret_cast<g1_xyzz*>(l.gathered.p);
        if (m->world == 1) B200_CUDA(cudaMemcpyAsync(gathered, l.partial.p, sizeof(g1_xyzz), cudaMemcpyDeviceToDevice, c.stream));
        B200_LAUNCH(k_sum_partials, 1, 32, 0, c.stream)(gathered, m->world, gathered + m->world);
        B200_CUDA(cudaGetLastError());
        if (i == 0) B200_CUDA(cudaMemcpyAsync(l.h_total.p, gathered + m->world, sizeof(g1_xyzz), cudaMemcpyDeviceToHost, c.stream));
        B200_CUDA(cudaEventRecord(l.done, c.stream));
    }
    for (size_t i = 0; i < nl; ++i) {
        B200_CUDA(cudaSetDevice(m->locals[i].ctx->c.device));
        B200_CUDA(cudaEventSynchronize(m->locals[i].done));
        if (b->end[i] > b->begin[i]) msm_collect_timing(&m->locals[i].ctx->c.msm, b->end[i] - b->begin[i], 1);
    }
    // 4. host: one inversion
    const g1_xyzz total = *reinterpret_cast<const g1_xyzz*>(m->locals[0].h_total.p);
    const g1_affine r = g1_to_affine(total);
    std::memcpy(out_xy, &r, 64);
    if (out_inf) *out_inf = g1_xyzz_is_inf(total) ? 1 : 0;
    return B200_OK;
}

int b200_multi_msm(b200_multi* m, const b200_multi_bases* bases, const uint64_t* scalars, size_t n, int scalars_montgomery,
                   uint64_t out_xy[8], int* out_is_identity) {
    B200_TRY
    if (!m || !bases || !scalars || !out_xy || n != bases->n) {
        set_error("multi_msm: null argument or n differs from the loaded bases");
        return B200_ERR_INVALID;
    }
    std::lock_guard<std::mutex> lk(m->mu);
    std::vector<const void*> slices(m->locals.size());
    for (size_t i = 0; i < slices.size(); ++i) slices[i] = scalars + 4 * bases->begin[i];
    return multi_msm(m, bases, slices.data(), 0, scalars_montgomery, out_xy, out_is_identity);
    B200_CATCH
}

int b200_multi_msm_local(b200_multi* m, const b200_multi_bases* bases, const void* const* scalars_local,
                         int scalars_on_device, int scalars_montgomery, uint64_t out_xy[8], int* out_is_identity) {
    B200_TRY
    if (!m || !bases || !scalars_local || !out_xy) return B200_ERR_INVALID;
    for (size_t i = 0; i < m->locals.size(); ++i)
        if (bases->end[i] > bases->begin[i] && !scalars_local[i]) return B200_ERR_INVALID;
    std::lock_guard<std::mutex> lk(m->mu);
    return multi_msm(m, bases, scalars_local, scalars_on_device ? 1 : 0, scalars_montgomery, out_xy, out_is_identity);
    B200_CATCH
}

}  // extern "C"
