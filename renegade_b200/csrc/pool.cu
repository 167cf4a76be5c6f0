// Prover pool: a FIFO job queue drained by N worker threads, each owning one context (stream +
// scratch) on the same device.  It is the device-side counterpart of the reference's
// `NativeProofManager` (crates/workers/proof-manager/src/implementations/native_proof_manager.rs:
// 138-201: a rayon pool fed with `spawn_fifo` from the job queue, one proof per worker): proving
// keys and SRS tables are shared read-only by all workers, so several proofs are in flight on one
// GPU and the latency-bound kernels of one proof (bucket reductions, scans, the host transcript)
// overlap the throughput-bound kernels of the others.  Verification jobs (b200verifyjobs.h) run the device verifiers
// on a worker's context in the same queue, so a caller that checks proofs on a proving GPU needs no context of its own.
// The express lane (b200express.h): a second queue that b200_pool_expedite moves a ticket's queued jobs to, drained by
// express workers whose contexts' streams outrank the normal workers' (and by normal workers when it backs up).
// Reserved SMs (b200reserved.h): the same pool with the express workers' contexts bound to a group of SMs of their own
// and the normal workers' to the rest, through green contexts (api.cu).
// Cancellation (b200cancel.h): a ticket's queued jobs are dropped from both queues; its running ones see their job's
// flag through b200::t_cancel, which the worker sets for the length of the call, and stop at their next abort point.
//
// Host-only code (std::thread) above the same C ABI the single-context entry points use.
#include <algorithm>
#include <condition_variable>
#include <deque>
#include <functional>
#include <map>
#include <memory>
#include <set>
#include <thread>
#include <vector>

#include "b200cancel.h"
#include "b200express.h"
#include "b200prover.h"
#include "b200reserved.h"
#include "b200settlement.h"
#include "b200verifyjobs.h"
#include "device_ctx.h"

namespace {

struct Bundle;

// The inputs a job copies at submit, so that the caller may free or reuse its own as soon as the submit returns.  Every
// copy is an allocation of its own: a pointer into one stays valid while more are taken, for as long as the job lives.
struct Held {
    std::vector<std::shared_ptr<void>> blocks;

    template <class T>
    T* copy(const T* src, size_t n) {  // nullptr for n == 0
        if (n == 0) return nullptr;
        std::shared_ptr<T> p(new T[n], std::default_delete<T[]>());
        std::copy(src, src + n, p.get());
        blocks.push_back(p);
        return p.get();
    }

    // A proof's inputs: public inputs (the key's num_inputs) and blinders
    b200_bundle_proof proof(b200_bundle_proof p) {
        p.pub_inputs = copy(p.pub_inputs, 4 * p.num_inputs);
        p.blinders = copy(p.blinders, 4 * 17);
        return p;
    }
    b200_bundle_witness proof(b200_bundle_witness p) {
        p.blinders = copy(p.blinders, 4 * 17);
        return p;
    }
    b200_link_item* link_items(const b200_link_item* its, size_t k) {
        b200_link_item* out = copy(its, k);
        for (size_t i = 0; i < k; ++i) {
            out[i].comm1 = copy(its[i].comm1, 8);
            out[i].comm2 = copy(its[i].comm2, 8);
        }
        return out;
    }
    b200_settlement_link* settlement_links(const b200_settlement_link* ls, size_t k) {
        b200_settlement_link* out = copy(ls, k);
        for (size_t i = 0; i < k; ++i) out[i].hint_comm = copy(ls[i].hint_comm, 8);
        return out;
    }
};

// A queued job: the context call it makes, on the copies it owns.  The call's captures point into `held`.
struct Job {
    uint64_t ticket = 0;
    std::shared_ptr<Bundle> bundle;  // set for the sub-jobs of a bundle (the bundle holds their ticket)
    Held held;
    std::function<int(b200_ctx*)> call;
    std::atomic<bool> cancel{false};  // set by a cancel while the job runs; the call reads it at its abort points
};

std::unique_ptr<Job> proof_job(const b200_bundle_proof& in) {
    std::unique_ptr<Job> j(new Job());
    const b200_bundle_proof p = j->held.proof(in);
    j->call = [p](b200_ctx* ctx) {
        return b200_plonk_prove(ctx, p.pk, p.wires, p.pub_inputs, p.blinders, p.proof, p.link_poly, nullptr);
    };
    return j;
}

std::unique_ptr<Job> proof_job(const b200_bundle_witness& in) {
    std::unique_ptr<Job> j(new Job());
    const b200_bundle_witness p = j->held.proof(in);
    j->call = [p](b200_ctx* ctx) {
        return b200_plonk_prove_witness(ctx, p.pk, p.witness, p.blinders, p.proof, p.link_poly, nullptr, p.pub_inputs_out);
    };
    return j;
}

// A single link stays on b200_plonk_link, which replays its CUDA graphs
std::unique_ptr<Job> link_job(const b200_bases* srs, const b200_link_item& it) {
    std::unique_ptr<Job> j(new Job());
    const b200_link_item x = *j->held.link_items(&it, 1);
    j->call = [srs, x](b200_ctx* ctx) {
        return b200_plonk_link(ctx, srs, x.a1, x.len1, x.a2, x.len2, x.comm1, x.comm2, x.alignment, x.offset, x.size, x.proof,
                               x.eta);
    };
    return j;
}

struct Done {
    int status = B200_OK;
    std::string message;
    uint64_t completed = 0;  // the pool's completed count right after the ticket's last job
    unsigned worker = 0;     // the worker that ran that job (express workers after the normal ones); kNoWorker: dropped
};
constexpr unsigned kNoWorker = ~0u;

Done cancelled_done() {
    Done d;
    d.status = B200_ERR_CANCELLED;
    d.message = "pool: the job was cancelled (B200_ERR_CANCELLED)";
    return d;
}

// A bundle: proofs first, then — once all of them are in — the link proofs between their wire-0 polynomials; one
// ticket for the whole thing.  Its links name proofs of the same bundle only; a settlement linked against hints kept from
// earlier proofs (the settlement arms of `NativeProofManager::handle_proof_job`, native_proof_manager.rs:514-660) is a
// settlement job, one call of b200_plonk_prove_settlement.
// Both bundle entry points (wire tables and witness vectors) share it: a link job needs only each proof's key, proof and
// link polynomial.
struct BundleHint {
    const b200_pk* pk;
    b200_proof* proof;
    uint64_t* link_poly;
};
struct Bundle {
    uint64_t ticket = 0;
    const b200_bases* srs = nullptr;
    std::vector<BundleHint> proofs;
    std::vector<b200_bundle_link> links;
    size_t pending = 0;     // sub-jobs of the current phase still queued or running
    bool linking = false;   // false: proof phase, true: link phase
    bool expedited = false; // its link jobs are forked onto the express queue
    bool cancelled = false; // forks no link jobs; finishes with B200_ERR_CANCELLED once its running sub-jobs are out
    Done result;            // first failure wins (a cancel overrides it)
};

}  // namespace

// Two queues: the normal one, FIFO in submit order, and the express queue, FIFO in the order jobs were expedited.  Workers
// 0..n_normal-1 take from the express queue when it holds more jobs than there are idle express workers, else from the
// normal queue; the express workers (n_normal and up, each with an express context) take from the express queue only.
struct b200_pool {
    std::vector<b200_ctx*> ctxs;     // the normal workers' contexts, then the express workers'
    unsigned n_normal = 0;
    unsigned sms[2] = {0, 0};        // SMs of the normal and the express group (b200_pool_create_reserved); 0, 0: no partition
    std::vector<std::thread> workers;
    std::mutex mu;
    std::condition_variable cv_job, cv_express, cv_done;  // cv_job: normal workers, cv_express: express workers
    std::deque<std::unique_ptr<Job>> queue, express;
    std::vector<Job*> running;       // per worker: the job it runs, or nullptr
    unsigned idle_express = 0;       // express workers running no job (and not yet gone at shutdown)
    std::map<uint64_t, Done> done;   // finished, not yet waited for
    std::set<uint64_t> inflight;     // queued or running
    std::map<uint64_t, Bundle*> bundles;  // unfinished bundles by ticket, so that expediting one marks it
    uint64_t next_ticket = 1;
    uint64_t n_submitted = 0, n_completed = 0, n_failed = 0, n_running = 0;
    bool stopping = false;

    static std::unique_ptr<Job> make_link_job(const std::shared_ptr<Bundle>& b, const b200_bundle_link& l) {
        const BundleHint& pa = b->proofs[l.a];
        const BundleHint& pb = b->proofs[l.b];
        // comm1 / comm2: the `linking_wire_comm` of each hint
        std::unique_ptr<Job> j = link_job(b->srs, {pa.link_poly, ((size_t)1 << b200_pk_log_n(pa.pk)) + 2, pb.link_poly,
                                                   ((size_t)1 << b200_pk_log_n(pb.pk)) + 2, pa.proof->wires_poly_comms[0],
                                                   pb.proof->wires_poly_comms[0], l.alignment, l.offset, l.size, l.proof, nullptr});
        j->ticket = b->ticket;
        j->bundle = b;
        return j;
    }

    // The queue worker w takes its next job from: &express, &queue, or nullptr (none for it now)
    std::deque<std::unique_ptr<Job>>* source(unsigned w) {
        if (w >= n_normal) return express.empty() ? nullptr : &express;
        if (express.size() > idle_express) return &express;
        return queue.empty() ? nullptr : &queue;
    }

    // A bundle whose last sub-job is out (finished with `last`, or dropped): its ticket is done.  Caller holds mu.
    void finish_bundle(Bundle& b, const Done& last) {
        b.result.completed = last.completed;
        b.result.worker = last.worker;
        bundles.erase(b.ticket);
        inflight.erase(b.ticket);
        done.emplace(b.ticket, b.result);
    }

    // Cancels the jobs of `ticket`, or of every ticket with `all`: drops the queued ones (each counts as completed and
    // failed) and flags the running ones.  Caller holds mu.  Returns how many it dropped.
    size_t cancel(uint64_t ticket, bool all) {
        auto hit = [&](const Job& j) { return all || j.ticket == ticket; };
        for (auto& kv : bundles)
            if (all || kv.first == ticket) {
                kv.second->cancelled = true;  // no link jobs from now on, and the ticket's status is the cancel
                kv.second->result = cancelled_done();
            }
        for (Job* j : running)
            if (j && hit(*j)) j->cancel = true;
        std::vector<std::unique_ptr<Job>> gone;
        for (std::deque<std::unique_ptr<Job>>* q : {&queue, &express}) {
            std::deque<std::unique_ptr<Job>> rest;
            for (std::unique_ptr<Job>& j : *q) {
                if (hit(*j)) gone.push_back(std::move(j));
                else rest.push_back(std::move(j));
            }
            q->swap(rest);
        }
        for (std::unique_ptr<Job>& j : gone) {
            ++n_completed;
            ++n_failed;
            Done d = cancelled_done();
            d.completed = n_completed;
            d.worker = kNoWorker;
            if (!j->bundle) {
                inflight.erase(j->ticket);
                done.emplace(j->ticket, std::move(d));
            } else if (--j->bundle->pending == 0) {
                finish_bundle(*j->bundle, d);
            }
        }
        return gone.size();
    }

    void notify_jobs(bool to_express) {
        if (to_express) cv_express.notify_all();
        cv_job.notify_all();  // a normal worker takes an express job no idle express worker will
    }

    void run(unsigned w) {
        const bool is_express = w >= n_normal;
        std::condition_variable& cv = is_express ? cv_express : cv_job;
        for (;;) {
            std::unique_ptr<Job> job;
            {
                std::unique_lock<std::mutex> lk(mu);
                std::deque<std::unique_ptr<Job>>* q = nullptr;
                cv.wait(lk, [&] { return (q = source(w)) != nullptr || stopping; });
                if (!q) {  // stopping and drained
                    if (is_express) {
                        --idle_express;  // gone: a normal worker takes what a bundle forks onto the express queue from now
                        lk.unlock();
                        cv_job.notify_all();
                    }
                    return;
                }
                job = std::move(q->front());
                q->pop_front();
                ++n_running;
                if (is_express) --idle_express;
                running[w] = job.get();
            }
            Done d;
            b200::t_cancel = &job->cancel;
            d.status = job->call(ctxs[w]);
            b200::t_cancel = nullptr;
            if (d.status != B200_OK) d.message = b200_last_error();  // this worker's thread-local message
            bool new_jobs = false, new_express = false;
            {
                std::lock_guard<std::mutex> lk(mu);
                running[w] = nullptr;
                --n_running;
                if (is_express) ++idle_express;
                ++n_completed;
                if (d.status != B200_OK) ++n_failed;
                d.completed = n_completed;
                d.worker = w;
                if (!job->bundle) {
                    inflight.erase(job->ticket);
                    done.emplace(job->ticket, std::move(d));
                } else {
                    Bundle& b = *job->bundle;
                    if (d.status != B200_OK && b.result.status == B200_OK) b.result = d;
                    if (--b.pending == 0) {
                        if (!b.linking && b.result.status == B200_OK && !b.links.empty()) {
                            b.linking = true;  // every proof is in: fork the link proofs
                            std::deque<std::unique_ptr<Job>>& q = b.expedited ? express : queue;
                            for (const b200_bundle_link& l : b.links) q.push_back(make_link_job(job->bundle, l));
                            b.pending = b.links.size();
                            n_submitted += b.links.size();
                            new_jobs = true;
                            new_express = b.expedited;
                        } else {
                            finish_bundle(b, d);
                        }
                    }
                }
            }
            if (new_jobs) notify_jobs(new_express);
            cv_done.notify_all();
        }
    }
};

// Queues jobs[0..n) under one new ticket: a single job, or the proof jobs of `bundle`.  Nothing is queued on a refusal.
static int pool_push(b200_pool* pool, std::unique_ptr<Job>* jobs, size_t n, const std::shared_ptr<Bundle>& bundle,
                     uint64_t* ticket) {
    {
        std::lock_guard<std::mutex> lk(pool->mu);
        if (pool->stopping) {
            b200::set_error("pool: shutting down");
            return B200_ERR_INVALID;
        }
        const uint64_t t = pool->next_ticket++;
        *ticket = t;
        if (bundle) {
            bundle->ticket = t;
            bundle->pending = n;
            pool->bundles.emplace(t, bundle.get());
        }
        pool->n_submitted += n;
        pool->inflight.insert(t);
        for (size_t i = 0; i < n; ++i) {
            jobs[i]->ticket = t;
            jobs[i]->bundle = bundle;
            pool->queue.push_back(std::move(jobs[i]));
        }
    }
    if (n == 1)
        pool->cv_job.notify_one();
    else
        pool->cv_job.notify_all();
    return B200_OK;
}

static int push_one(b200_pool* pool, std::unique_ptr<Job> job, uint64_t* ticket) {
    return pool_push(pool, &job, 1, nullptr, ticket);
}

// A bundle submission after its NULL-handle checks, for both entry points: check each proof entry and the links against the
// proofs, then queue one proof job per entry under one ticket.  Nothing is queued on a refusal.
template <class P>
static int bundle_push(b200_pool* pool, const char* who, const b200_bases* srs, const P* proofs, size_t n_proofs,
                       const b200_bundle_link* links, size_t n_links, uint64_t* ticket) {
    for (size_t i = 0; i < n_proofs; ++i) {
        const int rc = b200::check_entry(proofs[i], std::string(who) + ": proof " + std::to_string(i));
        if (rc != B200_OK) return rc;
    }
    for (size_t i = 0; i < n_links; ++i) {
        const b200_bundle_link& l = links[i];
        if (l.a >= n_proofs || l.b >= n_proofs || !l.proof || !proofs[l.a].link_poly || !proofs[l.b].link_poly)
            return b200::refuse(std::string(who) + ": a link names a proof that is missing or has no link_poly buffer");
    }
    std::shared_ptr<Bundle> b(new Bundle());
    b->srs = srs;
    b->links.assign(links, links + n_links);
    std::vector<std::unique_ptr<Job>> jobs;
    for (size_t i = 0; i < n_proofs; ++i) {
        b->proofs.push_back({proofs[i].pk, proofs[i].proof, proofs[i].link_poly});
        jobs.push_back(proof_job(proofs[i]));
    }
    return pool_push(pool, jobs.data(), jobs.size(), b, ticket);
}

// A pool of n_workers normal and n_express express workers; with `groups`, the express workers' contexts on groups[0] and
// the normal workers' on groups[1].  Nothing is left behind on a failure.
static int pool_create(int device, unsigned n_workers, unsigned n_express, const b200::SmGroup* groups, b200_pool** out) {
    std::unique_ptr<b200_pool> p(new b200_pool());
    for (unsigned i = 0; i < n_workers + n_express; ++i) {
        b200_ctx* c = nullptr;
        const bool express = i >= n_workers;
        const int rc = b200::context_create(device, express, groups ? &groups[express ? 0 : 1] : nullptr, &c);
        if (rc != B200_OK) {
            for (b200_ctx* q : p->ctxs) b200_shutdown(q);
            return rc;
        }
        p->ctxs.push_back(c);
    }
    p->n_normal = n_workers;
    p->idle_express = n_express;
    p->running.assign(p->ctxs.size(), nullptr);
    if (groups) {
        p->sms[0] = groups[1].sms;
        p->sms[1] = groups[0].sms;
    }
    b200_pool* raw = p.release();
    for (unsigned i = 0; i < n_workers + n_express; ++i) raw->workers.emplace_back([raw, i] { raw->run(i); });
    *out = raw;
    return B200_OK;
}

extern "C" {

int b200_pool_create(int device, unsigned n_workers, b200_pool** out) { return b200_pool_create_express(device, n_workers, 0, out); }

int b200_pool_create_express(int device, unsigned n_workers, unsigned n_express, b200_pool** out) {
    B200_TRY
    if (!out || n_workers == 0 || n_workers > 64 || n_express > 64) {
        b200::set_error("pool: n_workers must be in [1, 64] and n_express in [0, 64]");
        return B200_ERR_INVALID;
    }
    return pool_create(device, n_workers, n_express, nullptr, out);
    B200_CATCH
}

int b200_pool_create_reserved(int device, unsigned n_workers, unsigned n_express, unsigned express_sms, b200_pool** out) {
    B200_TRY
    const char* bad = !out                                   ? "null out"
                      : n_workers == 0 || n_workers > 64     ? "n_workers must be in [1, 64]"
                      : n_express == 0 || n_express > 64     ? "n_express must be in [1, 64]: the reserved SMs are the express workers'"
                      : express_sms == 0 || express_sms % 8  ? "express_sms must be a positive multiple of 8 (the SM granularity of a split)"
                      : express_sms > 248                    ? "express_sms must leave at least 8 SMs for the normal group (at most 248)"
                                                             : nullptr;
    if (bad) {
        b200::set_error(std::string("pool_create_reserved: ") + bad);
        return B200_ERR_INVALID;
    }
    b200::SmGroup groups[2];
    const int rc = b200::sm_split(device, express_sms, groups);
    if (rc != B200_OK) {
        b200::set_error("pool_create_reserved: " + std::string(b200_last_error()));
        return rc;
    }
    return pool_create(device, n_workers, n_express, groups, out);
    B200_CATCH
}

int b200_pool_partition(const b200_pool* pool, unsigned out[2]) {
    if (!pool || !out) {
        b200::set_error("pool_partition: null argument");
        return B200_ERR_INVALID;
    }
    out[0] = pool->sms[0];
    out[1] = pool->sms[1];
    return B200_OK;
}

int b200_pool_probe_sms(b200_pool* pool, unsigned worker, uint64_t mask[4]) {
    B200_TRY
    if (!pool || !mask || worker >= pool->ctxs.size()) {
        b200::set_error("pool_probe_sms: null pool or mask, or a worker index out of range");
        return B200_ERR_INVALID;
    }
    for (int i = 0; i < 4; ++i) mask[i] = 0;
    b200::Context& c = pool->ctxs[worker]->c;
    std::lock_guard<std::mutex> lk(c.mu);
    return b200::probe_sms(&c, mask);
    B200_CATCH
}

void b200_pool_destroy(b200_pool* pool) {
    if (!pool) return;
    {
        std::lock_guard<std::mutex> lk(pool->mu);
        pool->stopping = true;  // workers drain what is queued, then leave
    }
    pool->cv_job.notify_all();
    pool->cv_express.notify_all();
    for (std::thread& t : pool->workers) t.join();
    for (b200_ctx* c : pool->ctxs) b200_shutdown(c);
    delete pool;
}

unsigned b200_pool_workers(const b200_pool* pool) { return pool ? pool->n_normal : 0u; }

b200_ctx* b200_pool_ctx(b200_pool* pool, unsigned worker) {
    if (!pool || worker >= pool->n_normal) return nullptr;  // express contexts are the pool's own
    return pool->ctxs[worker];
}

int b200_pool_submit_prove(b200_pool* pool, const b200_pk* pk, const uint64_t* wires,
                           const uint64_t* pub_inputs, size_t num_inputs, const uint64_t* blinders,
                           b200_proof* proof, uint64_t* link_poly, uint64_t* ticket) {
    B200_TRY
    if (!pool || !pk || !ticket) return b200::refuse("pool_submit_prove: null argument");
    const b200_bundle_proof p{pk, wires, pub_inputs, num_inputs, blinders, proof, link_poly};
    const int rc = b200::check_entry(p, "pool_submit_prove");
    return rc != B200_OK ? rc : push_one(pool, proof_job(p), ticket);
    B200_CATCH
}

int b200_pool_submit_prove_witness(b200_pool* pool, const b200_pk* pk, const uint64_t* witness, const uint64_t* blinders,
                                   b200_proof* proof, uint64_t* link_poly, uint64_t* pub_inputs_out, uint64_t* ticket) {
    B200_TRY
    if (!pool || !pk || !ticket) return b200::refuse("pool_submit_prove_witness: null argument");
    const b200_bundle_witness p{pk, witness, blinders, proof, link_poly, pub_inputs_out};
    const int rc = b200::check_entry(p, "pool_submit_prove_witness");
    return rc != B200_OK ? rc : push_one(pool, proof_job(p), ticket);
    B200_CATCH
}

int b200_pool_submit_prove_batch(b200_pool* pool, const b200_pk* pk, const b200_prove_item* items, size_t k, int* statuses,
                                 uint64_t* ticket) {
    B200_TRY
    if (!pool || !pk || (k && !items) || !ticket) return b200::refuse("pool_submit_prove_batch: null argument");
    for (size_t i = 0; i < k; ++i) {
        const int rc = b200::check_prove_item(pk, items[i], "pool_submit_prove_batch: item " + std::to_string(i));
        if (rc != B200_OK) return rc;
    }
    const size_t ni = b200_pk_num_inputs(pk);
    std::unique_ptr<Job> j(new Job());
    b200_prove_item* its = j->held.copy(items, k);
    for (size_t i = 0; i < k; ++i) {
        its[i].pub_inputs = j->held.copy(items[i].pub_inputs, 4 * ni);
        its[i].blinders = j->held.copy(items[i].blinders, 4 * 17);
    }
    j->call = [pk, its, k, statuses](b200_ctx* ctx) { return b200_plonk_prove_batch(ctx, pk, its, k, statuses); };
    return push_one(pool, std::move(j), ticket);
    B200_CATCH
}

int b200_pool_submit_prove_witness_batch(b200_pool* pool, const b200_pk* pk, const b200_witness_item* items, size_t k,
                                         int* statuses, uint64_t* ticket) {
    B200_TRY
    if (!pool || !pk || (k && !items) || !ticket) return b200::refuse("pool_submit_prove_witness_batch: null argument");
    int rc = b200::check_wiring(pk, "pool_submit_prove_witness_batch");  // a batch of no items is refused too
    if (rc != B200_OK) return rc;
    for (size_t i = 0; i < k; ++i)
        if ((rc = b200::check_witness_item(pk, items[i], "pool_submit_prove_witness_batch: item " + std::to_string(i))) != B200_OK)
            return rc;
    std::unique_ptr<Job> j(new Job());
    b200_witness_item* its = j->held.copy(items, k);
    for (size_t i = 0; i < k; ++i) its[i].blinders = j->held.copy(items[i].blinders, 4 * 17);
    j->call = [pk, its, k, statuses](b200_ctx* ctx) { return b200_plonk_prove_witness_batch(ctx, pk, its, k, statuses); };
    return push_one(pool, std::move(j), ticket);
    B200_CATCH
}

int b200_pool_submit_link(b200_pool* pool, const b200_bases* srs, const uint64_t* a1, size_t len1,
                          const uint64_t* a2, size_t len2, const uint64_t* comm1, const uint64_t* comm2,
                          unsigned alignment, size_t offset, size_t size, b200_link_proof* proof,
                          uint64_t* ticket) {
    B200_TRY
    if (!pool || !srs || !ticket) return b200::refuse("pool_submit_link: null argument");
    const b200_link_item x{a1, len1, a2, len2, comm1, comm2, alignment, offset, size, proof, nullptr};
    const int rc = b200::check_link_ptrs(x, "pool_submit_link");
    return rc != B200_OK ? rc : push_one(pool, link_job(srs, x), ticket);
    B200_CATCH
}

int b200_pool_submit_link_batch(b200_pool* pool, const b200_bases* srs, const b200_link_item* items, size_t k,
                                int* statuses, uint64_t* ticket) {
    B200_TRY
    if (!pool || !srs || (k && !items) || !ticket) return b200::refuse("pool_submit_link_batch: null argument");
    for (size_t i = 0; i < k; ++i) {
        const int rc = b200::check_link_ptrs(items[i], "pool_submit_link_batch: item " + std::to_string(i));
        if (rc != B200_OK) return rc;
    }
    std::unique_ptr<Job> j(new Job());
    const b200_link_item* its = j->held.link_items(items, k);
    j->call = [srs, its, k, statuses](b200_ctx* ctx) { return b200_plonk_link_batch(ctx, srs, its, k, statuses); };
    return push_one(pool, std::move(j), ticket);
    B200_CATCH
}

int b200_pool_submit_bundle(b200_pool* pool, const b200_bases* srs, const b200_bundle_proof* proofs, size_t n_proofs,
                            const b200_bundle_link* links, size_t n_links, uint64_t* ticket) {
    B200_TRY
    if (!pool || !proofs || n_proofs == 0 || (n_links && (!links || !srs)) || !ticket)
        return b200::refuse("pool_submit_bundle: null argument");
    return bundle_push(pool, "pool_submit_bundle", srs, proofs, n_proofs, links, n_links, ticket);
    B200_CATCH
}

int b200_pool_submit_bundle_witness(b200_pool* pool, const b200_bases* srs, const b200_bundle_witness* proofs,
                                    size_t n_proofs, const b200_bundle_link* links, size_t n_links, uint64_t* ticket) {
    B200_TRY
    if (!pool || !proofs || n_proofs == 0 || (n_links && (!links || !srs)) || !ticket)
        return b200::refuse("pool_submit_bundle_witness: null argument");
    return bundle_push(pool, "pool_submit_bundle_witness", srs, proofs, n_proofs, links, n_links, ticket);
    B200_CATCH
}

int b200_pool_submit_settlement(b200_pool* pool, const b200_bases* srs, const b200_bundle_proof* proof,
                                const b200_settlement_link* links, size_t n_links, int* statuses, uint64_t* ticket) {
    B200_TRY
    const char* who = "pool_submit_settlement";
    if (!pool || !proof || !ticket) return b200::refuse(std::string(who) + ": null argument");
    const int rc = b200::settlement_check(srs, *proof, links, n_links, who);
    if (rc != B200_OK) return rc;
    std::unique_ptr<Job> j(new Job());
    const b200_bundle_proof p = j->held.proof(*proof);
    const b200_settlement_link* ls = j->held.settlement_links(links, n_links);
    j->call = [srs, p, ls, n_links, statuses](b200_ctx* ctx) {
        return b200_plonk_prove_settlement(ctx, srs, p.pk, p.wires, p.pub_inputs, p.blinders, p.proof, p.link_poly, ls, n_links,
                                           statuses);
    };
    return push_one(pool, std::move(j), ticket);
    B200_CATCH
}

int b200_pool_submit_settlement_witness(b200_pool* pool, const b200_bases* srs, const b200_bundle_witness* proof,
                                        const b200_settlement_link* links, size_t n_links, int* statuses, uint64_t* ticket) {
    B200_TRY
    const char* who = "pool_submit_settlement_witness";
    if (!pool || !proof || !ticket) return b200::refuse(std::string(who) + ": null argument");
    const int rc = b200::settlement_check(srs, *proof, links, n_links, who);
    if (rc != B200_OK) return rc;
    std::unique_ptr<Job> j(new Job());
    const b200_bundle_witness p = j->held.proof(*proof);
    const b200_settlement_link* ls = j->held.settlement_links(links, n_links);
    j->call = [srs, p, ls, n_links, statuses](b200_ctx* ctx) {
        return b200_plonk_prove_settlement_witness(ctx, srs, p.pk, p.witness, p.blinders, p.proof, p.link_poly, p.pub_inputs_out,
                                                   ls, n_links, statuses);
    };
    return push_one(pool, std::move(j), ticket);
    B200_CATCH
}

int b200_pool_submit_verify(b200_pool* pool, int mode, const b200_verifying_key* vks, size_t n_vks, const b200_batch_proof* proofs,
                            size_t n_proofs, const b200_batch_link* links, size_t n_links, const uint64_t g2_h[16],
                            const uint64_t g2_tau_h[16], int* all_accepted, uint8_t* verdicts, uint64_t* ticket) {
    B200_TRY
    const char* who = "pool_submit_verify";
    // what the verifiers' own checks (b200::verify_check) do not cover, then theirs: nothing is copied before both pass
    const char* bad = !pool                                                      ? "null pool"
                      : !ticket                                                  ? "null ticket"
                      : mode != 0 && mode != 1                                   ? "mode must be 0 or 1"
                      : n_vks && !vks                                            ? "null vks with n_vks > 0"
                      : n_proofs && !proofs                                      ? "null proofs with n_proofs > 0"
                      : n_links && !links                                        ? "null links with n_links > 0"
                      : !g2_h || !g2_tau_h                                       ? "null G2 record"
                      : n_proofs + n_links && !verdicts                          ? "null verdicts with items to verify"
                      : n_vks > 0xffffffffu || n_proofs + n_links > 0xffffffffu ? "more than 2^32 - 1 keys or items"
                                                                                 : nullptr;
    if (bad) {
        b200::set_error(std::string(who) + ": " + bad);
        return B200_ERR_INVALID;
    }
    // before any copy: the copy of a proof's public inputs reads vks[proofs[i].vk]
    const int rc = b200::verify_check(who, vks, n_vks, proofs, n_proofs, links, n_links, g2_h, g2_tau_h);
    if (rc != B200_OK) return rc;
    std::unique_ptr<Job> j(new Job());
    Held& h = j->held;
    b200_verifying_key* v = h.copy(vks, n_vks);
    for (size_t i = 0; i < n_vks; ++i) {
        v[i].k = h.copy(vks[i].k, 20);
        v[i].selector_comms = h.copy(vks[i].selector_comms, 104);
        v[i].sigma_comms = h.copy(vks[i].sigma_comms, 40);
    }
    b200_batch_proof* p = h.copy(proofs, n_proofs);
    for (size_t i = 0; i < n_proofs; ++i) {
        p[i].pub_inputs = h.copy(proofs[i].pub_inputs, 4 * vks[proofs[i].vk].num_inputs);
        p[i].proof = h.copy(proofs[i].proof, 1);
    }
    b200_batch_link* l = h.copy(links, n_links);
    for (size_t i = 0; i < n_links; ++i) {
        l[i].comm1 = h.copy(links[i].comm1, 8);
        l[i].comm2 = h.copy(links[i].comm2, 8);
        l[i].proof = h.copy(links[i].proof, 1);
    }
    const uint64_t* g2 = h.copy(g2_h, 16);
    const uint64_t* g2_tau = h.copy(g2_tau_h, 16);
    j->call = [=](b200_ctx* ctx) {  // mode 0: b200_plonk_verify_each, 1: b200_plonk_batch_verify
        if (mode == 0) return b200_plonk_verify_each(ctx, v, n_vks, p, n_proofs, l, n_links, g2, g2_tau, verdicts);
        int all = 0;
        const int st = b200_plonk_batch_verify(ctx, v, n_vks, p, n_proofs, l, n_links, g2, g2_tau, &all, verdicts);
        if (all_accepted) *all_accepted = all;
        return st;
    };
    return push_one(pool, std::move(j), ticket);
    B200_CATCH
}

int b200_pool_expedite(b200_pool* pool, uint64_t ticket, size_t* moved) {
    B200_TRY
    if (!pool || !moved || ticket == 0) {
        b200::set_error("pool_expedite: null pool or moved, or ticket 0");
        return B200_ERR_INVALID;
    }
    size_t n = 0;
    {
        std::lock_guard<std::mutex> lk(pool->mu);
        if (ticket >= pool->next_ticket) {
            b200::set_error("pool_expedite: unknown ticket");
            return B200_ERR_INVALID;
        }
        if (!pool->inflight.count(ticket) && !pool->done.count(ticket)) {
            b200::set_error("pool_expedite: ticket already waited for");
            return B200_ERR_INVALID;
        }
        auto b = pool->bundles.find(ticket);
        if (b != pool->bundles.end()) b->second->expedited = true;  // the links it forks later go to the express queue
        std::deque<std::unique_ptr<Job>> rest;
        for (std::unique_ptr<Job>& j : pool->queue) {
            if (j->ticket == ticket) {
                pool->express.push_back(std::move(j));
                ++n;
            } else {
                rest.push_back(std::move(j));
            }
        }
        pool->queue.swap(rest);
    }
    *moved = n;
    if (n) pool->notify_jobs(true);
    return B200_OK;
    B200_CATCH
}

// b200_pool_cancel and b200_pool_cancel_all (all = true, ticket unused)
static int pool_cancel(b200_pool* pool, uint64_t ticket, bool all, size_t* dropped, const char* who) {
    if (!pool || !dropped || (!all && ticket == 0)) {
        b200::set_error(std::string(who) + ": null pool or dropped, or ticket 0");
        return B200_ERR_INVALID;
    }
    size_t n = 0;
    {
        std::lock_guard<std::mutex> lk(pool->mu);
        if (!all && ticket >= pool->next_ticket) {
            b200::set_error(std::string(who) + ": unknown ticket");
            return B200_ERR_INVALID;
        }
        if (!all && !pool->inflight.count(ticket) && !pool->done.count(ticket)) {
            b200::set_error(std::string(who) + ": ticket already waited for");
            return B200_ERR_INVALID;
        }
        n = pool->cancel(ticket, all);
    }
    *dropped = n;
    if (n) pool->cv_done.notify_all();  // waits on the dropped tickets, and b200_pool_wait_all
    return B200_OK;
}

int b200_pool_cancel(b200_pool* pool, uint64_t ticket, size_t* dropped) {
    B200_TRY
    return pool_cancel(pool, ticket, false, dropped, "pool_cancel");
    B200_CATCH
}

int b200_pool_cancel_all(b200_pool* pool, size_t* dropped) {
    B200_TRY
    return pool_cancel(pool, 0, true, dropped, "pool_cancel_all");
    B200_CATCH
}

// b200_pool_wait, and with info != nullptr the ticket's completion index and worker
static int pool_wait(b200_pool* pool, uint64_t ticket, uint64_t* info, const char* who) {
    if (!pool || ticket == 0) {
        b200::set_error(std::string(who) + ": bad ticket");
        return B200_ERR_INVALID;
    }
    std::unique_lock<std::mutex> lk(pool->mu);
    if (ticket >= pool->next_ticket) {
        b200::set_error(std::string(who) + ": unknown ticket");
        return B200_ERR_INVALID;
    }
    for (;;) {
        auto it = pool->done.find(ticket);
        if (it != pool->done.end()) {
            const Done d = std::move(it->second);
            pool->done.erase(it);
            lk.unlock();
            if (info) {
                info[0] = d.completed;
                info[1] = d.worker;
            }
            if (d.status != B200_OK) b200::set_error(d.message);
            return d.status;
        }
        if (!pool->inflight.count(ticket)) {
            b200::set_error(std::string(who) + ": ticket already waited for");
            return B200_ERR_INVALID;
        }
        pool->cv_done.wait(lk);
    }
}

int b200_pool_wait(b200_pool* pool, uint64_t ticket) {
    B200_TRY
    return pool_wait(pool, ticket, nullptr, "pool_wait");
    B200_CATCH
}

int b200_pool_wait_info(b200_pool* pool, uint64_t ticket, uint64_t info[2]) {
    B200_TRY
    if (!info) {
        b200::set_error("pool_wait_info: null info");
        return B200_ERR_INVALID;
    }
    return pool_wait(pool, ticket, info, "pool_wait_info");
    B200_CATCH
}

int b200_pool_wait_all(b200_pool* pool) {
    B200_TRY
    if (!pool) {
        b200::set_error("pool_wait_all: null pool");
        return B200_ERR_INVALID;
    }
    std::unique_lock<std::mutex> lk(pool->mu);
    pool->cv_done.wait(lk, [&] { return pool->queue.empty() && pool->express.empty() && pool->n_running == 0; });
    int status = B200_OK;
    std::string message;
    for (auto& kv : pool->done)  // tickets are increasing: report the oldest failure
        if (kv.second.status != B200_OK && status == B200_OK) {
            status = kv.second.status;
            message = kv.second.message;
        }
    pool->done.clear();
    lk.unlock();
    if (status != B200_OK) b200::set_error(message);
    return status;
    B200_CATCH
}

int b200_pool_stats(b200_pool* pool, uint64_t out[4]) {
    if (!pool || !out) {
        b200::set_error("pool_stats: null argument");
        return B200_ERR_INVALID;
    }
    std::lock_guard<std::mutex> lk(pool->mu);
    out[0] = pool->n_submitted;
    out[1] = pool->n_completed;
    out[2] = pool->n_failed;
    out[3] = pool->queue.size() + pool->express.size();
    return B200_OK;
}

}  // extern "C"

// ---------------------------------------------------------------------------------------------------------------
// The whole box behind one object: one prover pool per device, the SRS tables and proving keys replicated on every
// device (whole proofs do not shard: SURVEY.md §8(e) "independent jobs => replicas, one proof stream per GPU, no
// communication"), each job routed to the device with the fewest unfinished jobs.  What a single Rust host process
// (the relayer's `NativeProofManager`) needs to use all GPUs without managing devices itself.
// ---------------------------------------------------------------------------------------------------------------
struct b200_box {
    std::vector<int> devices;
    std::vector<b200_pool*> pools;
};
struct b200_box_srs {
    std::vector<b200_bases*> per_dev;
    const b200_box* owner = nullptr;  // the box that made it
};
struct b200_box_pk {
    std::vector<b200_pk*> per_dev;
    const b200_box* owner = nullptr;  // the box that made it
};

namespace {
constexpr int kBoxTicketShift = 48;  // ticket = device index << 48 | the device pool's ticket

// ordinal >= 0: only the box entries on that CUDA device are candidates
int box_least_loaded(b200_box* box, int ordinal = -1) {
    int best = 0;
    uint64_t best_load = ~0ull;
    for (size_t i = 0; i < box->pools.size(); ++i) {
        if (ordinal >= 0 && box->devices[i] != ordinal) continue;
        uint64_t st[4];
        if (b200_pool_stats(box->pools[i], st) != B200_OK) continue;
        const uint64_t load = st[0] - st[1];  // submitted - completed
        if (load < best_load) {
            best_load = load;
            best = (int)i;
        }
    }
    return best;
}

// The box entry a job reading ws[0..n) (witness vectors, wire tables, hint polynomials) runs on: a pointer into device
// memory pins the job to that device (the least loaded of the box entries with its ordinal); host, pinned and managed
// memory can be read from any device.  Refused: a device outside the box, or device pointers on two different devices.
int box_witness_device(b200_box* box, const char* who, const uint64_t* const* ws, size_t n, int* out) {
    int ordinal = -1;
    for (size_t i = 0; i < n; ++i) {
        cudaPointerAttributes a{};
        if (cudaPointerGetAttributes(&a, ws[i]) != cudaSuccess) {
            cudaGetLastError();  // a pointer CUDA does not know is ordinary host memory
            continue;
        }
        if (a.type != cudaMemoryTypeDevice) continue;
        if (ordinal >= 0 && a.device != ordinal) {
            b200::set_error(std::string(who) + ": the witnesses lie on two devices (" + std::to_string(ordinal) + " and " +
                            std::to_string(a.device) + "); a bundle or settlement runs on one");
            return B200_ERR_INVALID;
        }
        ordinal = a.device;
    }
    if (ordinal >= 0 && std::find(box->devices.begin(), box->devices.end(), ordinal) == box->devices.end()) {
        b200::set_error(std::string(who) + ": the witness lies on device " + std::to_string(ordinal) + ", which is not in the box");
        return B200_ERR_INVALID;
    }
    *out = box_least_loaded(box, ordinal);
    return B200_OK;
}

// A key or SRS this box made.  One made by another box holds memory of that box's contexts, even when both boxes have as
// many devices.
template <class T>
bool box_owns(const b200_box* box, const T* x) {
    return x && x->owner == box && x->per_dev.size() == box->pools.size();
}

// Runs submit(box->pools[d], &t) and returns the box ticket: d << kBoxTicketShift | t
template <class Submit>
int box_submit(b200_box* box, int d, uint64_t* ticket, Submit submit) {
    uint64_t t = 0;
    const int rc = submit(box->pools[d], &t);
    if (rc != B200_OK) return rc;
    *ticket = ((uint64_t)d << kBoxTicketShift) | t;
    return B200_OK;
}

// Every proof of a bundle with its box key: all keys (and the SRS, if any) must be this box's
int box_bundle_check(const b200_box* box, const char* who, const b200_box_srs* srs, const b200_box_pk* const* pks, size_t n) {
    if (srs && !box_owns(box, srs)) {
        b200::set_error(std::string(who) + ": SRS of another box");
        return B200_ERR_INVALID;
    }
    for (size_t i = 0; i < n; ++i)
        if (!box_owns(box, pks[i])) {
            b200::set_error(std::string(who) + ": proof " + std::to_string(i) + " has no key or a key of another box");
            return B200_ERR_INVALID;
        }
    return B200_OK;
}

// One key per device, made by make(device's first context, device's SRS, &key) from the same arguments
template <class Make>
int box_replicate(b200_box* box, const char* who, const b200_box_srs* srs, b200_box_pk** out, Make make) {
    if (!box || !out || !box_owns(box, srs)) {
        b200::set_error(std::string(who) + ": null argument or SRS of another box");
        return B200_ERR_INVALID;
    }
    std::unique_ptr<b200_box_pk> pk(new b200_box_pk());
    pk->per_dev.assign(box->pools.size(), nullptr);
    pk->owner = box;
    for (size_t i = 0; i < box->pools.size(); ++i) {
        const int rc = make(b200_pool_ctx(box->pools[i], 0), srs->per_dev[i], &pk->per_dev[i]);
        if (rc != B200_OK) {
            b200_box_pk_free(box, pk.release());
            return rc;
        }
    }
    *out = pk.release();
    return B200_OK;
}
}  // namespace

extern "C" {

void b200_box_destroy(b200_box* box) {
    if (!box) return;
    for (b200_pool* p : box->pools) b200_pool_destroy(p);
    delete box;
}

int b200_box_create(const int* devices, int n_dev, unsigned workers_per_device, b200_box** out) {
    return b200_box_create_express(devices, n_dev, workers_per_device, 0, out);
}

}  // extern "C"

// A box of one pool per device, each made by make(device, &pool); nothing is left behind on a failure
template <class Make>
static int box_create(const int* devices, int n_dev, b200_box** out, Make make) {
    if (!devices || n_dev <= 0 || n_dev > 64 || !out) {
        b200::set_error("box_create: need 1..64 device ordinals");
        return B200_ERR_INVALID;
    }
    std::unique_ptr<b200_box> box(new b200_box());
    for (int i = 0; i < n_dev; ++i) {
        b200_pool* p = nullptr;
        const int rc = make(devices[i], &p);
        if (rc != B200_OK) {
            b200_box_destroy(box.release());
            return rc;
        }
        box->devices.push_back(devices[i]);
        box->pools.push_back(p);
    }
    *out = box.release();
    return B200_OK;
}

extern "C" {

int b200_box_create_express(const int* devices, int n_dev, unsigned workers_per_device, unsigned express_per_device,
                            b200_box** out) {
    B200_TRY
    return box_create(devices, n_dev, out, [&](int device, b200_pool** p) {
        return b200_pool_create_express(device, workers_per_device, express_per_device, p);
    });
    B200_CATCH
}

int b200_box_create_reserved(const int* devices, int n_dev, unsigned workers_per_device, unsigned express_per_device,
                             unsigned express_sms, b200_box** out) {
    B200_TRY
    return box_create(devices, n_dev, out, [&](int device, b200_pool** p) {
        return b200_pool_create_reserved(device, workers_per_device, express_per_device, express_sms, p);
    });
    B200_CATCH
}

int b200_box_devices(const b200_box* box) { return box ? (int)box->pools.size() : 0; }
b200_pool* b200_box_pool(b200_box* box, int i) {
    if (!box || i < 0 || i >= (int)box->pools.size()) return nullptr;
    return box->pools[i];
}

void b200_box_srs_free(b200_box* box, b200_box_srs* srs) {
    if (!srs) return;
    for (size_t i = 0; i < srs->per_dev.size(); ++i)
        if (srs->per_dev[i]) b200_bases_free(box && i < box->pools.size() ? b200_pool_ctx(box->pools[i], 0) : nullptr, srs->per_dev[i]);
    delete srs;
}

int b200_box_srs_load(b200_box* box, const uint8_t* points64, size_t n, int window_bits, int check_on_curve, b200_box_srs** out) {
    B200_TRY
    if (!box || !points64 || !out) return B200_ERR_INVALID;
    std::unique_ptr<b200_box_srs> s(new b200_box_srs());
    s->per_dev.assign(box->pools.size(), nullptr);
    s->owner = box;
    for (size_t i = 0; i < box->pools.size(); ++i) {
        // the on-curve assertion of srs.rs:178-179 once is enough: every device gets the same bytes
        const int rc = b200_bases_load(b200_pool_ctx(box->pools[i], 0), points64, n, window_bits, i == 0 ? check_on_curve : 0, &s->per_dev[i]);
        if (rc != B200_OK) {
            b200_box_srs_free(box, s.release());
            return rc;
        }
    }
    *out = s.release();
    return B200_OK;
    B200_CATCH
}

void b200_box_pk_free(b200_box* box, b200_box_pk* pk) {
    if (!pk) return;
    for (size_t i = 0; i < pk->per_dev.size(); ++i)
        if (pk->per_dev[i]) b200_pk_free(box && i < box->pools.size() ? b200_pool_ctx(box->pools[i], 0) : nullptr, pk->per_dev[i]);
    delete pk;
}

int b200_box_preprocess(b200_box* box, const b200_box_srs* srs, unsigned log_n, size_t num_inputs, const uint64_t* selectors_evals,
                        const uint64_t* perm, const uint64_t* k, b200_box_pk** out) {
    B200_TRY
    return box_replicate(box, "box_preprocess", srs, out, [&](b200_ctx* ctx, const b200_bases* s, b200_pk** pk) {
        return b200_plonk_preprocess(ctx, s, log_n, num_inputs, selectors_evals, perm, k, pk);
    });
    B200_CATCH
}

int b200_box_pk_verifying_key(const b200_box_pk* pk, uint64_t* selector_comms, uint64_t* sigma_comms) {
    if (!pk || pk->per_dev.empty()) return B200_ERR_INVALID;
    return b200_pk_verifying_key(pk->per_dev[0], selector_comms, sigma_comms);  // identical on every device
}

int b200_box_submit_prove(b200_box* box, const b200_box_pk* pk, const uint64_t* wires, const uint64_t* pub_inputs, size_t num_inputs,
                          const uint64_t* blinders, b200_proof* proof, uint64_t* link_poly, uint64_t* ticket) {
    B200_TRY
    if (!box || !ticket || !box_owns(box, pk)) {
        b200::set_error("box_submit_prove: null argument or key of another box");
        return B200_ERR_INVALID;
    }
    const int d = box_least_loaded(box);
    return box_submit(box, d, ticket, [&](b200_pool* p, uint64_t* t) {
        return b200_pool_submit_prove(p, pk->per_dev[d], wires, pub_inputs, num_inputs, blinders, proof, link_poly, t);
    });
    B200_CATCH
}

int b200_box_submit_bundle(b200_box* box, const b200_box_srs* srs, const b200_box_pk* const* pks, const b200_bundle_proof* proofs,
                           size_t n_proofs, const b200_bundle_link* links, size_t n_links, uint64_t* ticket) {
    B200_TRY
    if (!box || !pks || !proofs || n_proofs == 0 || !ticket || (n_links && !srs)) {
        b200::set_error("box_submit_bundle: null argument");
        return B200_ERR_INVALID;
    }
    const int rc = box_bundle_check(box, "box_submit_bundle", srs, pks, n_proofs);
    if (rc != B200_OK) return rc;
    const int d = box_least_loaded(box);  // a bundle stays on one device: its link proofs need its proofs' polynomials
    std::vector<b200_bundle_proof> local(proofs, proofs + n_proofs);
    for (size_t i = 0; i < n_proofs; ++i) local[i].pk = pks[i]->per_dev[d];
    return box_submit(box, d, ticket, [&](b200_pool* p, uint64_t* t) {
        return b200_pool_submit_bundle(p, srs ? srs->per_dev[d] : nullptr, local.data(), n_proofs, links, n_links, t);
    });
    B200_CATCH
}

int b200_box_preprocess_wiring(b200_box* box, const b200_box_srs* srs, unsigned log_n, size_t num_inputs,
                               const uint64_t* selectors_evals, const unsigned* wire_vars, size_t num_vars, const uint64_t* k,
                               b200_box_pk** out) {
    B200_TRY
    return box_replicate(box, "box_preprocess_wiring", srs, out, [&](b200_ctx* ctx, const b200_bases* s, b200_pk** pk) {
        return b200_plonk_preprocess_wiring(ctx, s, log_n, num_inputs, selectors_evals, wire_vars, num_vars, k, pk);
    });
    B200_CATCH
}

int b200_box_submit_prove_witness(b200_box* box, const b200_box_pk* pk, const uint64_t* witness, const uint64_t* blinders,
                                  b200_proof* proof, uint64_t* link_poly, uint64_t* pub_inputs_out, uint64_t* ticket) {
    B200_TRY
    if (!box || !witness || !ticket || !box_owns(box, pk)) {
        b200::set_error("box_submit_prove_witness: null argument or key of another box");
        return B200_ERR_INVALID;
    }
    int d = 0;
    const int rc = box_witness_device(box, "box_submit_prove_witness", &witness, 1, &d);
    if (rc != B200_OK) return rc;
    return box_submit(box, d, ticket, [&](b200_pool* p, uint64_t* t) {
        return b200_pool_submit_prove_witness(p, pk->per_dev[d], witness, blinders, proof, link_poly, pub_inputs_out, t);
    });
    B200_CATCH
}

int b200_box_submit_bundle_witness(b200_box* box, const b200_box_srs* srs, const b200_box_pk* const* pks,
                                   const b200_bundle_witness* proofs, size_t n_proofs, const b200_bundle_link* links,
                                   size_t n_links, uint64_t* ticket) {
    B200_TRY
    const char* who = "box_submit_bundle_witness";
    if (!box || !pks || !proofs || n_proofs == 0 || !ticket || (n_links && !srs)) {
        b200::set_error(std::string(who) + ": null argument");
        return B200_ERR_INVALID;
    }
    int rc = box_bundle_check(box, who, srs, pks, n_proofs);
    if (rc != B200_OK) return rc;
    std::vector<const uint64_t*> ws(n_proofs);
    for (size_t i = 0; i < n_proofs; ++i) {
        if (!proofs[i].witness) {
            b200::set_error(std::string(who) + ": proof " + std::to_string(i) + " has no witness");
            return B200_ERR_INVALID;
        }
        ws[i] = proofs[i].witness;
    }
    int d = 0;  // a bundle stays on one device: its link proofs need its proofs' polynomials
    rc = box_witness_device(box, who, ws.data(), n_proofs, &d);
    if (rc != B200_OK) return rc;
    std::vector<b200_bundle_witness> local(proofs, proofs + n_proofs);
    for (size_t i = 0; i < n_proofs; ++i) local[i].pk = pks[i]->per_dev[d];
    return box_submit(box, d, ticket, [&](b200_pool* p, uint64_t* t) {
        return b200_pool_submit_bundle_witness(p, srs ? srs->per_dev[d] : nullptr, local.data(), n_proofs, links, n_links, t);
    });
    B200_CATCH
}

// The device a box settlement runs on: its input (wire table or witness) and every hint polynomial count
static int box_settlement_device(b200_box* box, const char* who, const b200_box_srs* srs, const b200_box_pk* pk,
                                 const uint64_t* input, const b200_settlement_link* links, size_t n_links, int* out) {
    if (!box_owns(box, pk) || !box_owns(box, srs) || !input || (n_links && !links)) {
        b200::set_error(std::string(who) + ": null argument, or a key or SRS of another box");
        return B200_ERR_INVALID;
    }
    std::vector<const uint64_t*> ptrs{input};
    for (size_t i = 0; i < n_links; ++i)
        if (links[i].hint_poly) ptrs.push_back(links[i].hint_poly);  // a NULL one is refused by the pool's checks
    return box_witness_device(box, who, ptrs.data(), ptrs.size(), out);
}

int b200_box_submit_settlement(b200_box* box, const b200_box_srs* srs, const b200_box_pk* pk, const b200_bundle_proof* proof,
                               const b200_settlement_link* links, size_t n_links, int* statuses, uint64_t* ticket) {
    B200_TRY
    if (!box || !proof || !ticket) {
        b200::set_error("box_submit_settlement: null argument");
        return B200_ERR_INVALID;
    }
    int d = 0;
    const int rc = box_settlement_device(box, "box_submit_settlement", srs, pk, proof->wires, links, n_links, &d);
    if (rc != B200_OK) return rc;
    b200_bundle_proof local = *proof;
    local.pk = pk->per_dev[d];
    return box_submit(box, d, ticket, [&](b200_pool* p, uint64_t* t) {
        return b200_pool_submit_settlement(p, srs->per_dev[d], &local, links, n_links, statuses, t);
    });
    B200_CATCH
}

int b200_box_submit_settlement_witness(b200_box* box, const b200_box_srs* srs, const b200_box_pk* pk,
                                       const b200_bundle_witness* proof, const b200_settlement_link* links, size_t n_links,
                                       int* statuses, uint64_t* ticket) {
    B200_TRY
    if (!box || !proof || !ticket) {
        b200::set_error("box_submit_settlement_witness: null argument");
        return B200_ERR_INVALID;
    }
    int d = 0;
    const int rc = box_settlement_device(box, "box_submit_settlement_witness", srs, pk, proof->witness, links, n_links, &d);
    if (rc != B200_OK) return rc;
    b200_bundle_witness local = *proof;
    local.pk = pk->per_dev[d];
    return box_submit(box, d, ticket, [&](b200_pool* p, uint64_t* t) {
        return b200_pool_submit_settlement_witness(p, srs->per_dev[d], &local, links, n_links, statuses, t);
    });
    B200_CATCH
}

int b200_box_submit_verify(b200_box* box, int mode, const b200_verifying_key* vks, size_t n_vks, const b200_batch_proof* proofs,
                           size_t n_proofs, const b200_batch_link* links, size_t n_links, const uint64_t g2_h[16],
                           const uint64_t g2_tau_h[16], int* all_accepted, uint8_t* verdicts, uint64_t* ticket) {
    B200_TRY
    if (!box || !ticket) {
        b200::set_error("box_submit_verify: null box or ticket");
        return B200_ERR_INVALID;
    }
    // the job reads only its host copies: any device will do
    return box_submit(box, box_least_loaded(box), ticket, [&](b200_pool* p, uint64_t* t) {
        return b200_pool_submit_verify(p, mode, vks, n_vks, proofs, n_proofs, links, n_links, g2_h, g2_tau_h, all_accepted,
                                       verdicts, t);
    });
    B200_CATCH
}

// The pool of a box ticket's device and the ticket in that pool; nullptr for a NULL box or a device index out of range
static b200_pool* box_ticket_pool(b200_box* box, uint64_t ticket, const char* who, uint64_t* local) {
    const uint64_t d = ticket >> kBoxTicketShift;
    if (!box || d >= box->pools.size()) {
        b200::set_error(std::string(who) + ": bad ticket");
        return nullptr;
    }
    *local = ticket & (((uint64_t)1 << kBoxTicketShift) - 1);
    return box->pools[d];
}

int b200_box_wait(b200_box* box, uint64_t ticket) {
    B200_TRY
    uint64_t t = 0;
    b200_pool* p = box_ticket_pool(box, ticket, "box_wait", &t);
    return p ? b200_pool_wait(p, t) : B200_ERR_INVALID;
    B200_CATCH
}

int b200_box_expedite(b200_box* box, uint64_t ticket, size_t* moved) {
    B200_TRY
    uint64_t t = 0;
    b200_pool* p = box_ticket_pool(box, ticket, "box_expedite", &t);
    return p ? b200_pool_expedite(p, t, moved) : B200_ERR_INVALID;
    B200_CATCH
}

int b200_box_cancel(b200_box* box, uint64_t ticket, size_t* dropped) {
    B200_TRY
    uint64_t t = 0;
    b200_pool* p = box_ticket_pool(box, ticket, "box_cancel", &t);
    return p ? b200_pool_cancel(p, t, dropped) : B200_ERR_INVALID;
    B200_CATCH
}

int b200_box_cancel_all(b200_box* box, size_t* dropped) {
    B200_TRY
    if (!box || !dropped) {
        b200::set_error("box_cancel_all: null box or dropped");
        return B200_ERR_INVALID;
    }
    size_t total = 0;
    for (b200_pool* p : box->pools) {
        size_t n = 0;
        const int rc = b200_pool_cancel_all(p, &n);
        if (rc != B200_OK) return rc;
        total += n;
    }
    *dropped = total;
    return B200_OK;
    B200_CATCH
}

int b200_box_wait_info(b200_box* box, uint64_t ticket, uint64_t info[2]) {
    B200_TRY
    uint64_t t = 0;
    b200_pool* p = box_ticket_pool(box, ticket, "box_wait_info", &t);
    return p ? b200_pool_wait_info(p, t, info) : B200_ERR_INVALID;
    B200_CATCH
}

int b200_box_ticket_device(const b200_box* box, uint64_t ticket) {
    const uint64_t d = ticket >> kBoxTicketShift;
    return box && d < box->pools.size() ? (int)d : -1;
}

}  // extern "C"
