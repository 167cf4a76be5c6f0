// Prover pool: a FIFO job queue drained by N worker threads, each owning one context (stream +
// scratch) on the same device.  It is the device-side counterpart of the reference's
// `NativeProofManager` (crates/workers/proof-manager/src/implementations/native_proof_manager.rs:
// 138-201: a rayon pool fed with `spawn_fifo` from the job queue, one proof per worker): proving
// keys and SRS tables are shared read-only by all workers, so several proofs are in flight on one
// GPU and the latency-bound kernels of one proof (bucket reductions, scans, the host transcript)
// overlap the throughput-bound kernels of the others.  Verification jobs (b200verifyjobs.h) run the device verifiers
// on a worker's context in the same queue, so a caller that checks proofs on a proving GPU needs no context of its own.
//
// Host-only code (std::thread) above the same C ABI the single-context entry points use.
#include <algorithm>
#include <condition_variable>
#include <cstring>
#include <deque>
#include <map>
#include <memory>
#include <set>
#include <thread>
#include <vector>

#include "b200prover.h"
#include "b200settlement.h"
#include "b200verifyjobs.h"
#include "device_ctx.h"

namespace {

struct Bundle;

// The inputs of a verification job, copied at submit: the arrays with every pointer into the copies below, so the
// caller may free or reuse its own as soon as the submit returns.
struct VerifyCopy {
    int mode = 0;  // 0: b200_plonk_verify_each, 1: b200_plonk_batch_verify
    std::vector<b200_verifying_key> vks;
    std::vector<b200_batch_proof> proofs;
    std::vector<b200_batch_link> links;
    std::vector<uint64_t> limbs;  // each key's k / selector / sigma, each proof's public inputs, each link's comm1 / comm2
    std::vector<b200_proof> proof_bodies;
    std::vector<b200_link_proof> link_bodies;
    uint64_t g2_h[16], g2_tau_h[16];
    int* all_accepted = nullptr;  // the caller's outputs
    uint8_t* verdicts = nullptr;

    VerifyCopy(int m, const b200_verifying_key* v, size_t n_v, const b200_batch_proof* p, size_t n_p, const b200_batch_link* l,
               size_t n_l, const uint64_t* h, const uint64_t* tau_h)
        : mode(m), vks(v, v + n_v), proofs(p, p + n_p), links(l, l + n_l), proof_bodies(n_p), link_bodies(n_l) {
        size_t total = (20 + 104 + 40) * n_v + 16 * n_l;
        for (size_t i = 0; i < n_p; ++i) total += 4 * v[p[i].vk].num_inputs;
        limbs.resize(total);  // sized once: the pointers below stay valid
        uint64_t* at = limbs.data();
        auto take = [&at](const uint64_t* src, size_t n) {
            std::memcpy(at, src, 8 * n);
            const uint64_t* out = at;
            at += n;
            return out;
        };
        for (b200_verifying_key& vk : vks) {
            vk.k = take(vk.k, 20);
            vk.selector_comms = take(vk.selector_comms, 104);
            vk.sigma_comms = take(vk.sigma_comms, 40);
        }
        for (size_t i = 0; i < n_p; ++i) {
            const size_t ni = vks[proofs[i].vk].num_inputs;
            proofs[i].pub_inputs = ni ? take(proofs[i].pub_inputs, 4 * ni) : nullptr;
            proof_bodies[i] = *proofs[i].proof;
            proofs[i].proof = &proof_bodies[i];
        }
        for (size_t i = 0; i < n_l; ++i) {
            links[i].comm1 = take(links[i].comm1, 8);
            links[i].comm2 = take(links[i].comm2, 8);
            link_bodies[i] = *links[i].proof;
            links[i].proof = &link_bodies[i];
        }
        std::memcpy(g2_h, h, 128);
        std::memcpy(g2_tau_h, tau_h, 128);
    }

    int run(b200_ctx* ctx) const {
        if (mode == 0)
            return b200_plonk_verify_each(ctx, vks.data(), vks.size(), proofs.data(), proofs.size(), links.data(), links.size(),
                                          g2_h, g2_tau_h, verdicts);
        int all = 0;
        const int rc = b200_plonk_batch_verify(ctx, vks.data(), vks.size(), proofs.data(), proofs.size(), links.data(),
                                               links.size(), g2_h, g2_tau_h, &all, verdicts);
        if (all_accepted) *all_accepted = all;
        return rc;
    }
};

struct Job {
    enum Kind { kProve, kProveWitness, kProveBatch, kProveWitnessBatch, kLink, kLinkBatch, kSettlement, kSettlementWitness,
                kVerify } kind = kProve;
    uint64_t ticket = 0;
    // prove (wires: the table) and prove witness (wires: the witness vector)
    const b200_pk* pk = nullptr;
    const uint64_t* wires = nullptr;
    std::vector<uint64_t> pub_inputs, blinders;
    b200_proof* proof = nullptr;
    uint64_t* link_poly = nullptr;
    uint64_t* pub_inputs_out = nullptr;
    // prove batch: the items with pub_inputs / blinders pointing into the copies below (pub_inputs, blinders: k each)
    std::vector<b200_prove_item> items;
    // prove witness batch: the items with blinders pointing into the copies in `blinders` (k of them)
    std::vector<b200_witness_item> witness_items;
    int* statuses = nullptr;
    // link (one item) and link batch: the items with comm1 / comm2 pointing into the copies below (8 limbs each, two per
    // item)
    const b200_bases* srs = nullptr;
    std::vector<b200_link_item> link_items;
    std::vector<uint64_t> link_comms;
    std::shared_ptr<Bundle> bundle;  // set for the sub-jobs of a bundle (they carry no ticket of their own)
    // settlement (pk, wires, pub_inputs, blinders, proof, link_poly, pub_inputs_out, srs, statuses as above): the links
    // with hint_comm pointing into the copies in `link_comms` (8 limbs per link)
    std::vector<b200_settlement_link> settlement_links;
    // verify: everything the verifier reads, owned by the job
    std::unique_ptr<VerifyCopy> verify;

    void set_settlement_links(const b200_settlement_link* ls, size_t k) {  // the worker reads the copies
        settlement_links.assign(ls, ls + k);
        link_comms.resize(8 * k);
        for (size_t i = 0; i < k; ++i) {
            std::memcpy(&link_comms[8 * i], ls[i].hint_comm, 64);
            settlement_links[i].hint_comm = &link_comms[8 * i];
        }
    }

    void set_link_items(const b200_link_item* its, size_t k) {  // the worker reads the copies
        link_items.assign(its, its + k);
        link_comms.resize(16 * k);
        for (size_t i = 0; i < k; ++i) {
            std::memcpy(&link_comms[16 * i], its[i].comm1, 64);
            std::memcpy(&link_comms[16 * i + 8], its[i].comm2, 64);
            link_items[i].comm1 = &link_comms[16 * i];
            link_items[i].comm2 = &link_comms[16 * i + 8];
        }
    }
};

struct Done {
    int status = B200_OK;
    std::string message;
};

// A bundle: proofs first, then — once all of them are in — the link proofs between their wire-0 polynomials; one
// ticket for the whole thing.  Its links name proofs of the same bundle only; a settlement linked against hints kept from
// earlier proofs (the settlement arms of `NativeProofManager::handle_proof_job`, native_proof_manager.rs:514-660) is a
// settlement job (kSettlement), one call of b200_plonk_prove_settlement.
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
    Done result;            // first failure wins
};

}  // namespace

struct b200_pool {
    std::vector<b200_ctx*> ctxs;
    std::vector<std::thread> workers;
    std::mutex mu;
    std::condition_variable cv_job, cv_done;
    std::deque<std::unique_ptr<Job>> queue;
    std::map<uint64_t, Done> done;   // finished, not yet waited for
    std::set<uint64_t> inflight;     // queued or running
    uint64_t next_ticket = 1;
    uint64_t n_submitted = 0, n_completed = 0, n_failed = 0, n_running = 0;
    bool stopping = false;

    static std::unique_ptr<Job> make_link_job(const std::shared_ptr<Bundle>& b, const b200_bundle_link& l) {
        const BundleHint& pa = b->proofs[l.a];
        const BundleHint& pb = b->proofs[l.b];
        std::unique_ptr<Job> j(new Job());
        j->kind = Job::kLink;
        j->bundle = b;
        j->srs = b->srs;
        // comm1 / comm2: the `linking_wire_comm` of each hint
        const b200_link_item it{pa.link_poly, ((size_t)1 << b200_pk_log_n(pa.pk)) + 2, pb.link_poly,
                                ((size_t)1 << b200_pk_log_n(pb.pk)) + 2, pa.proof->wires_poly_comms[0], pb.proof->wires_poly_comms[0],
                                l.alignment, l.offset, l.size, l.proof, nullptr};
        j->set_link_items(&it, 1);
        return j;
    }

    void run(unsigned w) {
        for (;;) {
            std::unique_ptr<Job> job;
            {
                std::unique_lock<std::mutex> lk(mu);
                cv_job.wait(lk, [&] { return stopping || !queue.empty(); });
                if (queue.empty()) return;  // stopping and drained
                job = std::move(queue.front());
                queue.pop_front();
                ++n_running;
            }
            Done d;
            if (job->kind == Job::kProve) {
                d.status = b200_plonk_prove(ctxs[w], job->pk, job->wires,
                                            job->pub_inputs.empty() ? nullptr : job->pub_inputs.data(),
                                            job->blinders.data(), job->proof, job->link_poly, nullptr);
            } else if (job->kind == Job::kProveWitness) {
                d.status = b200_plonk_prove_witness(ctxs[w], job->pk, job->wires, job->blinders.data(), job->proof, job->link_poly,
                                                    nullptr, job->pub_inputs_out);
            } else if (job->kind == Job::kProveBatch) {
                d.status = b200_plonk_prove_batch(ctxs[w], job->pk, job->items.data(), job->items.size(), job->statuses);
            } else if (job->kind == Job::kProveWitnessBatch) {
                d.status = b200_plonk_prove_witness_batch(ctxs[w], job->pk, job->witness_items.data(), job->witness_items.size(),
                                                          job->statuses);
            } else if (job->kind == Job::kSettlement) {
                d.status = b200_plonk_prove_settlement(ctxs[w], job->srs, job->pk, job->wires,
                                                       job->pub_inputs.empty() ? nullptr : job->pub_inputs.data(),
                                                       job->blinders.data(), job->proof, job->link_poly,
                                                       job->settlement_links.data(), job->settlement_links.size(), job->statuses);
            } else if (job->kind == Job::kSettlementWitness) {
                d.status = b200_plonk_prove_settlement_witness(ctxs[w], job->srs, job->pk, job->wires, job->blinders.data(),
                                                               job->proof, job->link_poly, job->pub_inputs_out,
                                                               job->settlement_links.data(), job->settlement_links.size(),
                                                               job->statuses);
            } else if (job->kind == Job::kVerify) {
                d.status = job->verify->run(ctxs[w]);
            } else if (job->kind == Job::kLinkBatch) {
                d.status = b200_plonk_link_batch(ctxs[w], job->srs, job->link_items.data(), job->link_items.size(), job->statuses);
            } else {  // a single link stays on b200_plonk_link, which replays its CUDA graphs
                const b200_link_item& x = job->link_items[0];
                d.status = b200_plonk_link(ctxs[w], job->srs, x.a1, x.len1, x.a2, x.len2, x.comm1, x.comm2, x.alignment,
                                           x.offset, x.size, x.proof, x.eta);
            }
            if (d.status != B200_OK) d.message = b200_last_error();  // this worker's thread-local message
            bool new_jobs = false;
            {
                std::lock_guard<std::mutex> lk(mu);
                --n_running;
                ++n_completed;
                if (d.status != B200_OK) ++n_failed;
                if (!job->bundle) {
                    inflight.erase(job->ticket);
                    done.emplace(job->ticket, std::move(d));
                } else {
                    Bundle& b = *job->bundle;
                    if (d.status != B200_OK && b.result.status == B200_OK) b.result = d;
                    if (--b.pending == 0) {
                        if (!b.linking && b.result.status == B200_OK && !b.links.empty()) {
                            b.linking = true;  // every proof is in: fork the link proofs
                            for (const b200_bundle_link& l : b.links) queue.push_back(make_link_job(job->bundle, l));
                            b.pending = b.links.size();
                            n_submitted += b.links.size();
                            new_jobs = true;
                        } else {
                            inflight.erase(b.ticket);
                            done.emplace(b.ticket, b.result);
                        }
                    }
                }
            }
            if (new_jobs) cv_job.notify_all();
            cv_done.notify_all();
        }
    }
};

extern "C" {

int b200_pool_create(int device, unsigned n_workers, b200_pool** out) {
    B200_TRY
    if (!out || n_workers == 0 || n_workers > 64) {
        b200::set_error("pool: n_workers must be in [1, 64]");
        return B200_ERR_INVALID;
    }
    std::unique_ptr<b200_pool> p(new b200_pool());
    for (unsigned i = 0; i < n_workers; ++i) {
        b200_ctx* c = nullptr;
        const int rc = b200_init(device, &c);
        if (rc != B200_OK) {
            for (b200_ctx* q : p->ctxs) b200_shutdown(q);
            return rc;
        }
        p->ctxs.push_back(c);
    }
    b200_pool* raw = p.release();
    for (unsigned i = 0; i < n_workers; ++i) raw->workers.emplace_back([raw, i] { raw->run(i); });
    *out = raw;
    return B200_OK;
    B200_CATCH
}

void b200_pool_destroy(b200_pool* pool) {
    if (!pool) return;
    {
        std::lock_guard<std::mutex> lk(pool->mu);
        pool->stopping = true;  // workers drain what is queued, then leave
    }
    pool->cv_job.notify_all();
    for (std::thread& t : pool->workers) t.join();
    for (b200_ctx* c : pool->ctxs) b200_shutdown(c);
    delete pool;
}

unsigned b200_pool_workers(const b200_pool* pool) { return pool ? (unsigned)pool->ctxs.size() : 0u; }

b200_ctx* b200_pool_ctx(b200_pool* pool, unsigned worker) {
    if (!pool || worker >= pool->ctxs.size()) return nullptr;
    return pool->ctxs[worker];
}

static int pool_push(b200_pool* pool, std::unique_ptr<Job> job, uint64_t* ticket) {
    {
        std::lock_guard<std::mutex> lk(pool->mu);
        if (pool->stopping) {
            b200::set_error("pool: shutting down");
            return B200_ERR_INVALID;
        }
        job->ticket = pool->next_ticket++;
        *ticket = job->ticket;
        ++pool->n_submitted;
        pool->inflight.insert(job->ticket);
        pool->queue.push_back(std::move(job));
    }
    pool->cv_job.notify_one();
    return B200_OK;
}

int b200_pool_submit_prove(b200_pool* pool, const b200_pk* pk, const uint64_t* wires,
                           const uint64_t* pub_inputs, size_t num_inputs, const uint64_t* blinders,
                           b200_proof* proof, uint64_t* link_poly, uint64_t* ticket) {
    B200_TRY
    if (!pool || !pk || !wires || !blinders || !proof || !ticket || (num_inputs && !pub_inputs)) {
        b200::set_error("pool_submit_prove: null argument");
        return B200_ERR_INVALID;
    }
    if (num_inputs != b200_pk_num_inputs(pk)) {  // the worker reads exactly pk.num_inputs elements
        b200::set_error("pool_submit_prove: num_inputs does not match the proving key");
        return B200_ERR_INVALID;
    }
    std::unique_ptr<Job> j(new Job());
    j->kind = Job::kProve;
    j->pk = pk;
    j->wires = wires;
    j->pub_inputs.assign(pub_inputs, pub_inputs + 4 * num_inputs);
    j->blinders.assign(blinders, blinders + 4 * 17);
    j->proof = proof;
    j->link_poly = link_poly;
    return pool_push(pool, std::move(j), ticket);
    B200_CATCH
}

int b200_pool_submit_prove_witness(b200_pool* pool, const b200_pk* pk, const uint64_t* witness, const uint64_t* blinders,
                                   b200_proof* proof, uint64_t* link_poly, uint64_t* pub_inputs_out, uint64_t* ticket) {
    B200_TRY
    if (!pool || !pk || !witness || !blinders || !proof || !ticket) {
        b200::set_error("pool_submit_prove_witness: null argument");
        return B200_ERR_INVALID;
    }
    if (b200_pk_num_vars(pk) == 0) {
        b200::set_error("pool_submit_prove_witness: the key holds no wiring (made by b200_plonk_preprocess)");
        return B200_ERR_INVALID;
    }
    std::unique_ptr<Job> j(new Job());
    j->kind = Job::kProveWitness;
    j->pk = pk;
    j->wires = witness;
    j->blinders.assign(blinders, blinders + 4 * 17);
    j->proof = proof;
    j->link_poly = link_poly;
    j->pub_inputs_out = pub_inputs_out;
    return pool_push(pool, std::move(j), ticket);
    B200_CATCH
}

int b200_pool_submit_prove_batch(b200_pool* pool, const b200_pk* pk, const b200_prove_item* items, size_t k, int* statuses,
                                 uint64_t* ticket) {
    B200_TRY
    if (!pool || !pk || (k && !items) || !ticket) {
        b200::set_error("pool_submit_prove_batch: null argument");
        return B200_ERR_INVALID;
    }
    const size_t ni = b200_pk_num_inputs(pk);
    for (size_t i = 0; i < k; ++i)
        if (!items[i].wires || !items[i].blinders || !items[i].proof || (ni && !items[i].pub_inputs)) {
            b200::set_error("pool_submit_prove_batch: item " + std::to_string(i) + " has a NULL pointer");
            return B200_ERR_INVALID;
        }
    std::unique_ptr<Job> j(new Job());
    j->kind = Job::kProveBatch;
    j->pk = pk;
    j->statuses = statuses;
    j->pub_inputs.resize(4 * ni * k);
    j->blinders.resize(4 * 17 * k);
    j->items.assign(items, items + k);
    for (size_t i = 0; i < k; ++i) {  // the worker reads the copies
        if (ni) std::memcpy(&j->pub_inputs[4 * ni * i], items[i].pub_inputs, 32 * ni);
        std::memcpy(&j->blinders[4 * 17 * i], items[i].blinders, 32 * 17);
        j->items[i].pub_inputs = ni ? &j->pub_inputs[4 * ni * i] : nullptr;
        j->items[i].blinders = &j->blinders[4 * 17 * i];
    }
    return pool_push(pool, std::move(j), ticket);
    B200_CATCH
}

int b200_pool_submit_prove_witness_batch(b200_pool* pool, const b200_pk* pk, const b200_witness_item* items, size_t k,
                                         int* statuses, uint64_t* ticket) {
    B200_TRY
    if (!pool || !pk || (k && !items) || !ticket) {
        b200::set_error("pool_submit_prove_witness_batch: null argument");
        return B200_ERR_INVALID;
    }
    if (b200_pk_num_vars(pk) == 0) {
        b200::set_error("pool_submit_prove_witness_batch: the key holds no wiring (made by b200_plonk_preprocess)");
        return B200_ERR_INVALID;
    }
    for (size_t i = 0; i < k; ++i)
        if (!items[i].witness || !items[i].blinders || !items[i].proof) {
            b200::set_error("pool_submit_prove_witness_batch: item " + std::to_string(i) + " has a NULL pointer");
            return B200_ERR_INVALID;
        }
    std::unique_ptr<Job> j(new Job());
    j->kind = Job::kProveWitnessBatch;
    j->pk = pk;
    j->statuses = statuses;
    j->blinders.resize(4 * 17 * k);
    j->witness_items.assign(items, items + k);
    for (size_t i = 0; i < k; ++i) {  // the worker reads the copies
        std::memcpy(&j->blinders[4 * 17 * i], items[i].blinders, 32 * 17);
        j->witness_items[i].blinders = &j->blinders[4 * 17 * i];
    }
    return pool_push(pool, std::move(j), ticket);
    B200_CATCH
}

int b200_pool_submit_link(b200_pool* pool, const b200_bases* srs, const uint64_t* a1, size_t len1,
                          const uint64_t* a2, size_t len2, const uint64_t* comm1, const uint64_t* comm2,
                          unsigned alignment, size_t offset, size_t size, b200_link_proof* proof,
                          uint64_t* ticket) {
    B200_TRY
    if (!pool || !srs || !a1 || !a2 || !comm1 || !comm2 || !proof || !ticket) {
        b200::set_error("pool_submit_link: null argument");
        return B200_ERR_INVALID;
    }
    std::unique_ptr<Job> j(new Job());
    j->kind = Job::kLink;
    j->srs = srs;
    const b200_link_item it{a1, len1, a2, len2, comm1, comm2, alignment, offset, size, proof, nullptr};
    j->set_link_items(&it, 1);
    return pool_push(pool, std::move(j), ticket);
    B200_CATCH
}

int b200_pool_submit_link_batch(b200_pool* pool, const b200_bases* srs, const b200_link_item* items, size_t k,
                                int* statuses, uint64_t* ticket) {
    B200_TRY
    if (!pool || !srs || (k && !items) || !ticket) {
        b200::set_error("pool_submit_link_batch: null argument");
        return B200_ERR_INVALID;
    }
    for (size_t i = 0; i < k; ++i)
        if (!items[i].a1 || !items[i].a2 || !items[i].comm1 || !items[i].comm2 || !items[i].proof) {
            b200::set_error("pool_submit_link_batch: item " + std::to_string(i) + " has a NULL pointer");
            return B200_ERR_INVALID;
        }
    std::unique_ptr<Job> j(new Job());
    j->kind = Job::kLinkBatch;
    j->srs = srs;
    j->statuses = statuses;
    j->set_link_items(items, k);
    return pool_push(pool, std::move(j), ticket);
    B200_CATCH
}

// The part of a bundle submission both entry points share: check the links against the proofs' hints, then queue the
// proof jobs (each already filled in but for its `bundle`) under one ticket.  Nothing is queued on a refusal.
static int bundle_push(b200_pool* pool, const char* who, const b200_bases* srs, std::vector<BundleHint> hints,
                       const b200_bundle_link* links, size_t n_links, std::vector<std::unique_ptr<Job>> jobs, uint64_t* ticket) {
    for (size_t i = 0; i < n_links; ++i) {
        const b200_bundle_link& l = links[i];
        if (l.a >= hints.size() || l.b >= hints.size() || !l.proof || !hints[l.a].link_poly || !hints[l.b].link_poly) {
            b200::set_error(std::string(who) + ": a link names a proof that is missing or has no link_poly buffer");
            return B200_ERR_INVALID;
        }
    }
    std::shared_ptr<Bundle> b(new Bundle());
    b->srs = srs;
    b->proofs = std::move(hints);
    b->links.assign(links, links + n_links);
    b->pending = jobs.size();
    for (auto& j : jobs) j->bundle = b;
    {
        std::lock_guard<std::mutex> lk(pool->mu);
        if (pool->stopping) {
            b200::set_error("pool: shutting down");
            return B200_ERR_INVALID;
        }
        b->ticket = pool->next_ticket++;
        *ticket = b->ticket;
        pool->n_submitted += jobs.size();
        pool->inflight.insert(b->ticket);
        for (auto& j : jobs) pool->queue.push_back(std::move(j));
    }
    pool->cv_job.notify_all();
    return B200_OK;
}

int b200_pool_submit_bundle(b200_pool* pool, const b200_bases* srs, const b200_bundle_proof* proofs, size_t n_proofs,
                            const b200_bundle_link* links, size_t n_links, uint64_t* ticket) {
    B200_TRY
    if (!pool || !proofs || n_proofs == 0 || (n_links && (!links || !srs)) || !ticket) {
        b200::set_error("pool_submit_bundle: null argument");
        return B200_ERR_INVALID;
    }
    for (size_t i = 0; i < n_proofs; ++i) {
        const b200_bundle_proof& p = proofs[i];
        if (!p.pk || !p.wires || !p.blinders || !p.proof || (p.num_inputs && !p.pub_inputs) ||
            p.num_inputs != b200_pk_num_inputs(p.pk)) {
            b200::set_error("pool_submit_bundle: bad proof entry (null pointer or num_inputs does not match the key)");
            return B200_ERR_INVALID;
        }
    }
    std::vector<BundleHint> hints;
    std::vector<std::unique_ptr<Job>> jobs;
    for (size_t i = 0; i < n_proofs; ++i) {
        const b200_bundle_proof& p = proofs[i];
        hints.push_back({p.pk, p.proof, p.link_poly});
        std::unique_ptr<Job> j(new Job());
        j->kind = Job::kProve;
        j->pk = p.pk;
        j->wires = p.wires;
        j->pub_inputs.assign(p.pub_inputs, p.pub_inputs + 4 * p.num_inputs);
        j->blinders.assign(p.blinders, p.blinders + 4 * 17);
        j->proof = p.proof;
        j->link_poly = p.link_poly;
        jobs.push_back(std::move(j));
    }
    return bundle_push(pool, "pool_submit_bundle", srs, std::move(hints), links, n_links, std::move(jobs), ticket);
    B200_CATCH
}

int b200_pool_submit_bundle_witness(b200_pool* pool, const b200_bases* srs, const b200_bundle_witness* proofs,
                                    size_t n_proofs, const b200_bundle_link* links, size_t n_links, uint64_t* ticket) {
    B200_TRY
    if (!pool || !proofs || n_proofs == 0 || (n_links && (!links || !srs)) || !ticket) {
        b200::set_error("pool_submit_bundle_witness: null argument");
        return B200_ERR_INVALID;
    }
    for (size_t i = 0; i < n_proofs; ++i) {
        const b200_bundle_witness& p = proofs[i];
        if (!p.pk || !p.witness || !p.blinders || !p.proof) {
            b200::set_error("pool_submit_bundle_witness: proof " + std::to_string(i) + " has a NULL pointer");
            return B200_ERR_INVALID;
        }
        if (b200_pk_num_vars(p.pk) == 0) {
            b200::set_error("pool_submit_bundle_witness: the key of proof " + std::to_string(i) +
                            " holds no wiring (made by b200_plonk_preprocess)");
            return B200_ERR_INVALID;
        }
    }
    std::vector<BundleHint> hints;
    std::vector<std::unique_ptr<Job>> jobs;
    for (size_t i = 0; i < n_proofs; ++i) {
        const b200_bundle_witness& p = proofs[i];
        hints.push_back({p.pk, p.proof, p.link_poly});
        std::unique_ptr<Job> j(new Job());
        j->kind = Job::kProveWitness;
        j->pk = p.pk;
        j->wires = p.witness;
        j->blinders.assign(p.blinders, p.blinders + 4 * 17);
        j->proof = p.proof;
        j->link_poly = p.link_poly;
        j->pub_inputs_out = p.pub_inputs_out;
        jobs.push_back(std::move(j));
    }
    return bundle_push(pool, "pool_submit_bundle_witness", srs, std::move(hints), links, n_links, std::move(jobs), ticket);
    B200_CATCH
}

int b200_pool_submit_settlement(b200_pool* pool, const b200_bases* srs, const b200_bundle_proof* proof,
                                const b200_settlement_link* links, size_t n_links, int* statuses, uint64_t* ticket) {
    B200_TRY
    const char* who = "pool_submit_settlement";
    if (!pool || !proof || !ticket || !proof->pk || !proof->wires || !proof->blinders || !proof->proof ||
        (proof->num_inputs && !proof->pub_inputs)) {
        b200::set_error(std::string(who) + ": null argument");
        return B200_ERR_INVALID;
    }
    if (proof->num_inputs != b200_pk_num_inputs(proof->pk)) {  // the worker reads exactly pk.num_inputs elements
        b200::set_error(std::string(who) + ": num_inputs does not match the proving key");
        return B200_ERR_INVALID;
    }
    const int rc = b200::settlement_check(srs, proof->pk, /*witness=*/false, links, n_links, who);
    if (rc != B200_OK) return rc;
    std::unique_ptr<Job> j(new Job());
    j->kind = Job::kSettlement;
    j->srs = srs;
    j->pk = proof->pk;
    j->wires = proof->wires;
    j->pub_inputs.assign(proof->pub_inputs, proof->pub_inputs + 4 * proof->num_inputs);
    j->blinders.assign(proof->blinders, proof->blinders + 4 * 17);
    j->proof = proof->proof;
    j->link_poly = proof->link_poly;
    j->statuses = statuses;
    j->set_settlement_links(links, n_links);
    return pool_push(pool, std::move(j), ticket);
    B200_CATCH
}

int b200_pool_submit_settlement_witness(b200_pool* pool, const b200_bases* srs, const b200_bundle_witness* proof,
                                        const b200_settlement_link* links, size_t n_links, int* statuses, uint64_t* ticket) {
    B200_TRY
    const char* who = "pool_submit_settlement_witness";
    if (!pool || !proof || !ticket || !proof->pk || !proof->witness || !proof->blinders || !proof->proof) {
        b200::set_error(std::string(who) + ": null argument");
        return B200_ERR_INVALID;
    }
    const int rc = b200::settlement_check(srs, proof->pk, /*witness=*/true, links, n_links, who);
    if (rc != B200_OK) return rc;
    std::unique_ptr<Job> j(new Job());
    j->kind = Job::kSettlementWitness;
    j->srs = srs;
    j->pk = proof->pk;
    j->wires = proof->witness;
    j->blinders.assign(proof->blinders, proof->blinders + 4 * 17);
    j->proof = proof->proof;
    j->link_poly = proof->link_poly;
    j->pub_inputs_out = proof->pub_inputs_out;
    j->statuses = statuses;
    j->set_settlement_links(links, n_links);
    return pool_push(pool, std::move(j), ticket);
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
    const int rc = b200::verify_check(who, vks, n_vks, proofs, n_proofs, links, n_links, g2_h, g2_tau_h);
    if (rc != B200_OK) return rc;
    std::unique_ptr<Job> j(new Job());
    j->kind = Job::kVerify;
    j->verify.reset(new VerifyCopy(mode, vks, n_vks, proofs, n_proofs, links, n_links, g2_h, g2_tau_h));
    j->verify->all_accepted = all_accepted;
    j->verify->verdicts = verdicts;
    return pool_push(pool, std::move(j), ticket);
    B200_CATCH
}

int b200_pool_wait(b200_pool* pool, uint64_t ticket) {
    B200_TRY
    if (!pool || ticket == 0) {
        b200::set_error("pool_wait: bad ticket");
        return B200_ERR_INVALID;
    }
    std::unique_lock<std::mutex> lk(pool->mu);
    if (ticket >= pool->next_ticket) {
        b200::set_error("pool_wait: unknown ticket");
        return B200_ERR_INVALID;
    }
    for (;;) {
        auto it = pool->done.find(ticket);
        if (it != pool->done.end()) {
            const Done d = std::move(it->second);
            pool->done.erase(it);
            lk.unlock();
            if (d.status != B200_OK) b200::set_error(d.message);
            return d.status;
        }
        if (!pool->inflight.count(ticket)) {
            b200::set_error("pool_wait: ticket already waited for");
            return B200_ERR_INVALID;
        }
        pool->cv_done.wait(lk);
    }
    B200_CATCH
}

int b200_pool_wait_all(b200_pool* pool) {
    B200_TRY
    if (!pool) {
        b200::set_error("pool_wait_all: null pool");
        return B200_ERR_INVALID;
    }
    std::unique_lock<std::mutex> lk(pool->mu);
    pool->cv_done.wait(lk, [&] { return pool->queue.empty() && pool->n_running == 0; });
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
    out[3] = pool->queue.size();
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

bool box_owns(const b200_box* box, const b200_box_pk* pk) {
    return pk && pk->owner == box && pk->per_dev.size() == box->pools.size();
}
}  // namespace

extern "C" {

void b200_box_destroy(b200_box* box) {
    if (!box) return;
    for (b200_pool* p : box->pools) b200_pool_destroy(p);
    delete box;
}

int b200_box_create(const int* devices, int n_dev, unsigned workers_per_device, b200_box** out) {
    B200_TRY
    if (!devices || n_dev <= 0 || n_dev > 64 || !out) {
        b200::set_error("box_create: need 1..64 device ordinals");
        return B200_ERR_INVALID;
    }
    std::unique_ptr<b200_box> box(new b200_box());
    for (int i = 0; i < n_dev; ++i) {
        b200_pool* p = nullptr;
        const int rc = b200_pool_create(devices[i], workers_per_device, &p);
        if (rc != B200_OK) {
            b200_box_destroy(box.release());
            return rc;
        }
        box->devices.push_back(devices[i]);
        box->pools.push_back(p);
    }
    *out = box.release();
    return B200_OK;
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
    if (!box || !srs || !out || srs->per_dev.size() != box->pools.size()) return B200_ERR_INVALID;
    std::unique_ptr<b200_box_pk> pk(new b200_box_pk());
    pk->per_dev.assign(box->pools.size(), nullptr);
    pk->owner = box;
    for (size_t i = 0; i < box->pools.size(); ++i) {
        const int rc = b200_plonk_preprocess(b200_pool_ctx(box->pools[i], 0), srs->per_dev[i], log_n, num_inputs, selectors_evals, perm, k,
                                             &pk->per_dev[i]);
        if (rc != B200_OK) {
            b200_box_pk_free(box, pk.release());
            return rc;
        }
    }
    *out = pk.release();
    return B200_OK;
    B200_CATCH
}

int b200_box_pk_verifying_key(const b200_box_pk* pk, uint64_t* selector_comms, uint64_t* sigma_comms) {
    if (!pk || pk->per_dev.empty()) return B200_ERR_INVALID;
    return b200_pk_verifying_key(pk->per_dev[0], selector_comms, sigma_comms);  // identical on every device
}

int b200_box_submit_prove(b200_box* box, const b200_box_pk* pk, const uint64_t* wires, const uint64_t* pub_inputs, size_t num_inputs,
                          const uint64_t* blinders, b200_proof* proof, uint64_t* link_poly, uint64_t* ticket) {
    B200_TRY
    if (!box || !pk || !ticket || pk->per_dev.size() != box->pools.size()) {
        b200::set_error("box_submit_prove: null argument or key of another box");
        return B200_ERR_INVALID;
    }
    const int d = box_least_loaded(box);
    uint64_t t = 0;
    const int rc = b200_pool_submit_prove(box->pools[d], pk->per_dev[d], wires, pub_inputs, num_inputs, blinders, proof, link_poly, &t);
    if (rc != B200_OK) return rc;
    *ticket = ((uint64_t)d << kBoxTicketShift) | t;
    return B200_OK;
    B200_CATCH
}

int b200_box_submit_bundle(b200_box* box, const b200_box_srs* srs, const b200_box_pk* const* pks, const b200_bundle_proof* proofs,
                           size_t n_proofs, const b200_bundle_link* links, size_t n_links, uint64_t* ticket) {
    B200_TRY
    if (!box || !pks || !proofs || n_proofs == 0 || !ticket || (n_links && !srs)) {
        b200::set_error("box_submit_bundle: null argument");
        return B200_ERR_INVALID;
    }
    const int d = box_least_loaded(box);  // a bundle stays on one device: its link proofs need its proofs' polynomials
    std::vector<b200_bundle_proof> local(proofs, proofs + n_proofs);
    for (size_t i = 0; i < n_proofs; ++i) {
        if (!pks[i] || pks[i]->per_dev.size() != box->pools.size()) {
            b200::set_error("box_submit_bundle: missing key");
            return B200_ERR_INVALID;
        }
        local[i].pk = pks[i]->per_dev[d];
    }
    uint64_t t = 0;
    const int rc = b200_pool_submit_bundle(box->pools[d], srs ? srs->per_dev[d] : nullptr, local.data(), n_proofs, links, n_links, &t);
    if (rc != B200_OK) return rc;
    *ticket = ((uint64_t)d << kBoxTicketShift) | t;
    return B200_OK;
    B200_CATCH
}

int b200_box_preprocess_wiring(b200_box* box, const b200_box_srs* srs, unsigned log_n, size_t num_inputs,
                               const uint64_t* selectors_evals, const unsigned* wire_vars, size_t num_vars, const uint64_t* k,
                               b200_box_pk** out) {
    B200_TRY
    if (!box || !srs || !out || srs->per_dev.size() != box->pools.size()) {
        b200::set_error("box_preprocess_wiring: null argument or SRS of another box");
        return B200_ERR_INVALID;
    }
    std::unique_ptr<b200_box_pk> pk(new b200_box_pk());
    pk->per_dev.assign(box->pools.size(), nullptr);
    pk->owner = box;
    for (size_t i = 0; i < box->pools.size(); ++i) {
        const int rc = b200_plonk_preprocess_wiring(b200_pool_ctx(box->pools[i], 0), srs->per_dev[i], log_n, num_inputs,
                                                    selectors_evals, wire_vars, num_vars, k, &pk->per_dev[i]);
        if (rc != B200_OK) {
            b200_box_pk_free(box, pk.release());
            return rc;
        }
    }
    *out = pk.release();
    return B200_OK;
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
    int rc = box_witness_device(box, "box_submit_prove_witness", &witness, 1, &d);
    if (rc != B200_OK) return rc;
    uint64_t t = 0;
    rc = b200_pool_submit_prove_witness(box->pools[d], pk->per_dev[d], witness, blinders, proof, link_poly, pub_inputs_out, &t);
    if (rc != B200_OK) return rc;
    *ticket = ((uint64_t)d << kBoxTicketShift) | t;
    return B200_OK;
    B200_CATCH
}

int b200_box_submit_bundle_witness(b200_box* box, const b200_box_srs* srs, const b200_box_pk* const* pks,
                                   const b200_bundle_witness* proofs, size_t n_proofs, const b200_bundle_link* links,
                                   size_t n_links, uint64_t* ticket) {
    B200_TRY
    if (!box || !pks || !proofs || n_proofs == 0 || !ticket || (n_links && (!srs || srs->per_dev.size() != box->pools.size()))) {
        b200::set_error("box_submit_bundle_witness: null argument");
        return B200_ERR_INVALID;
    }
    std::vector<const uint64_t*> ws(n_proofs);
    for (size_t i = 0; i < n_proofs; ++i) {
        if (!box_owns(box, pks[i]) || !proofs[i].witness) {
            b200::set_error("box_submit_bundle_witness: proof " + std::to_string(i) + " has no witness or a key of another box");
            return B200_ERR_INVALID;
        }
        ws[i] = proofs[i].witness;
    }
    int d = 0;  // a bundle stays on one device: its link proofs need its proofs' polynomials
    int rc = box_witness_device(box, "box_submit_bundle_witness", ws.data(), n_proofs, &d);
    if (rc != B200_OK) return rc;
    std::vector<b200_bundle_witness> local(proofs, proofs + n_proofs);
    for (size_t i = 0; i < n_proofs; ++i) local[i].pk = pks[i]->per_dev[d];
    uint64_t t = 0;
    rc = b200_pool_submit_bundle_witness(box->pools[d], srs ? srs->per_dev[d] : nullptr, local.data(), n_proofs, links, n_links, &t);
    if (rc != B200_OK) return rc;
    *ticket = ((uint64_t)d << kBoxTicketShift) | t;
    return B200_OK;
    B200_CATCH
}

// The device a box settlement runs on: its input (wire table or witness) and every hint polynomial count
static int box_settlement_device(b200_box* box, const char* who, const b200_box_srs* srs, const b200_box_pk* pk,
                                 const uint64_t* input, const b200_settlement_link* links, size_t n_links, int* out) {
    if (!box_owns(box, pk) || !srs || srs->per_dev.size() != box->pools.size() || !input || (n_links && !links)) {
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
    int rc = box_settlement_device(box, "box_submit_settlement", srs, pk, proof->wires, links, n_links, &d);
    if (rc != B200_OK) return rc;
    b200_bundle_proof local = *proof;
    local.pk = pk->per_dev[d];
    uint64_t t = 0;
    rc = b200_pool_submit_settlement(box->pools[d], srs->per_dev[d], &local, links, n_links, statuses, &t);
    if (rc != B200_OK) return rc;
    *ticket = ((uint64_t)d << kBoxTicketShift) | t;
    return B200_OK;
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
    int rc = box_settlement_device(box, "box_submit_settlement_witness", srs, pk, proof->witness, links, n_links, &d);
    if (rc != B200_OK) return rc;
    b200_bundle_witness local = *proof;
    local.pk = pk->per_dev[d];
    uint64_t t = 0;
    rc = b200_pool_submit_settlement_witness(box->pools[d], srs->per_dev[d], &local, links, n_links, statuses, &t);
    if (rc != B200_OK) return rc;
    *ticket = ((uint64_t)d << kBoxTicketShift) | t;
    return B200_OK;
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
    const int d = box_least_loaded(box);  // the job reads only its host copies: any device will do
    uint64_t t = 0;
    const int rc = b200_pool_submit_verify(box->pools[d], mode, vks, n_vks, proofs, n_proofs, links, n_links, g2_h, g2_tau_h,
                                           all_accepted, verdicts, &t);
    if (rc != B200_OK) return rc;
    *ticket = ((uint64_t)d << kBoxTicketShift) | t;
    return B200_OK;
    B200_CATCH
}

int b200_box_wait(b200_box* box, uint64_t ticket) {
    B200_TRY
    const uint64_t d = ticket >> kBoxTicketShift;
    if (!box || d >= box->pools.size()) {
        b200::set_error("box_wait: bad ticket");
        return B200_ERR_INVALID;
    }
    return b200_pool_wait(box->pools[d], ticket & (((uint64_t)1 << kBoxTicketShift) - 1));
    B200_CATCH
}

int b200_box_ticket_device(const b200_box* box, uint64_t ticket) {
    const uint64_t d = ticket >> kBoxTicketShift;
    return box && d < box->pools.size() ? (int)d : -1;
}

}  // extern "C"
