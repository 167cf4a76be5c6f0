/* b200settlement.h — settlement jobs of libb200prover: a settlement statement proved and linked, in one call, against
 * the link hints a caller kept from earlier validity proofs.  The shape of every settlement arm of the reference's
 * `NativeProofManager::handle_proof_job` (native_proof_manager.rs:514-660): `singleprover_prove_with_hint`, then
 * `link_proofs(&hint, &settlement_hint, &layout)` for each hint the job brings.
 *
 * A job layer over the core ABI of b200prover.h (its prover, link batch, pool and box), declared in a header of its
 * own: b200prover.h stays the core entry-point set, and this header adds the six settlement entry points of the same
 * library (libb200prover.so), with the same conventions and error codes. */
#ifndef B200SETTLEMENT_H
#define B200SETTLEMENT_H

#include "b200prover.h"

#ifdef __cplusplus
extern "C" {
#endif

/* ---- on a context -------------------------------------------------------------------------------------------------- */
/* One link proof of a settlement: the caller's stored hint FIRST, the settlement proof's hint second
 * (`link_proofs(&validity_hint, &settlement_hint, &layout)`, intent_and_balance.rs:57-72, intent_only.rs:42-47). */
typedef struct {
    const uint64_t* hint_poly;   /* `linking_wire_poly`: hint_len x 4 limbs, Montgomery; host or device pointer */
    size_t hint_len;
    const uint64_t* hint_comm;   /* its `linking_wire_comm`, 8 limbs (host) */
    unsigned alignment; size_t offset; size_t size;   /* GroupLayout */
    b200_link_proof* proof;
    uint64_t* eta;               /* may be NULL */
} b200_settlement_link;
/* A settlement job in one call: the shape of every settlement arm of `NativeProofManager::handle_proof_job`
 * (native_proof_manager.rs:514-660: `singleprover_prove_with_hint`, then `link_proofs` against each hint the job brings).
 * Proves the statement as b200_plonk_prove (replaying its CUDA graphs once the key is warm), then makes all n_links link
 * proofs as ONE link batch (b200_plonk_link_batch's buffers), each between links[i]'s stored hint and the settlement's
 * link polynomial P, which the links read from device memory.
 * Bytes: proof and link_poly (may be NULL) are byte-identical to b200_plonk_prove's with the same inputs; link i's proof
 * and eta are byte-identical to b200_plonk_link(ctx, srs, hint_poly, hint_len, P, n + 2, hint_comm,
 * proof->wires_poly_comms[0], alignment, offset, size, ...).
 * statuses (may be NULL) receives n_links + 1 codes: statuses[0] the proof's, statuses[1 + i] link i's.
 *  - a settlement witness that does not satisfy the circuit: statuses[0] = B200_ERR_UNSATISFIED and no link proof is
 *    made; the proof and every link proof are zeroed, every link status is B200_ERR_UNSATISFIED, no eta is written;
 *  - a hint that differs from P on its group (a stale hint): that link's status is B200_ERR_UNSATISFIED and its proof is
 *    zeroed; every other link is still made.
 * Returns B200_OK when everything was made, else B200_ERR_UNSATISFIED; b200_last_error() says whether the proof failed or
 * which links did.  Argument errors return B200_ERR_INVALID before any device work (no kernel launched, no output
 * written) and the message names the link: everything b200_plonk_prove refuses, a NULL srs, a NULL links pointer with
 * n_links > 0, a link with a NULL hint_poly / hint_comm / proof, or one b200_plonk_link would refuse with len1 = hint_len
 * and len2 = n + 2 (size 0, size >= max length, alignment > 28, size > 2^alignment, a polynomial longer than the SRS).
 * n_links = 0 is a plain proof. */
int b200_plonk_prove_settlement(b200_ctx* ctx, const b200_bases* srs, const b200_pk* pk, const uint64_t* wires,
                                const uint64_t* pub_inputs, const uint64_t* blinders, b200_proof* proof, uint64_t* link_poly,
                                const b200_settlement_link* links, size_t n_links, int* statuses);
/* b200_plonk_prove_settlement from the settlement's witness vector, as b200_plonk_prove_witness: proof, link_poly and
 * pub_inputs_out (may be NULL) are byte-identical to its; links, statuses and return codes exactly as
 * b200_plonk_prove_settlement (B200_ERR_INVALID also for a key without wiring). */
int b200_plonk_prove_settlement_witness(b200_ctx* ctx, const b200_bases* srs, const b200_pk* pk, const uint64_t* witness,
                                        const uint64_t* blinders, b200_proof* proof, uint64_t* link_poly,
                                        uint64_t* pub_inputs_out, const b200_settlement_link* links, size_t n_links,
                                        int* statuses);

/* ---- on a prover pool ---------------------------------------------------------------------------------------------- */
/* Queue one `b200_plonk_prove_settlement(ctx_of_some_worker, srs, proof->pk, proof->wires, proof->pub_inputs,
 * proof->blinders, proof->proof, proof->link_poly, links, n_links, statuses)` as ONE job on one worker (one job in
 * b200_pool_stats).  The links array, each hint_comm, the blinders and the public inputs are copied at submit; the wire
 * table, the hint polynomials, every output buffer and statuses (may be NULL) stay owned by the caller until the ticket
 * has been waited for.  Every argument error of b200_plonk_prove_settlement (and proof->num_inputs differing from the
 * key's) is refused at submit with B200_ERR_INVALID and nothing is queued.  The ticket's status is the call's. */
int b200_pool_submit_settlement(b200_pool* pool, const b200_bases* srs, const b200_bundle_proof* proof,
                                const b200_settlement_link* links, size_t n_links, int* statuses, uint64_t* ticket);
/* b200_pool_submit_settlement with the settlement given as a witness vector: one b200_plonk_prove_settlement_witness
 * job; copies, ownership, refusals (also a key without wiring) and the ticket's status as b200_pool_submit_settlement. */
int b200_pool_submit_settlement_witness(b200_pool* pool, const b200_bases* srs, const b200_bundle_witness* proof,
                                        const b200_settlement_link* links, size_t n_links, int* statuses, uint64_t* ticket);

/* ---- on a box ------------------------------------------------------------------------------------------------------ */
/* b200_pool_submit_settlement on one device of the box: `pk` is the box key of the settlement (proof->pk is ignored),
 * srs a box SRS.  Every device-memory pointer of the job (the wire table and each hint polynomial) must lie on one
 * device of the box, and the job runs there (the least loaded of the box entries with that ordinal); a job with no
 * device pointers goes to the least-loaded device.  Refused at submit with B200_ERR_INVALID: pointers on two devices, a
 * device outside the box, a key or SRS of another box, and every refusal of b200_pool_submit_settlement. */
int b200_box_submit_settlement(b200_box* box, const b200_box_srs* srs, const b200_box_pk* pk, const b200_bundle_proof* proof,
                               const b200_settlement_link* links, size_t n_links, int* statuses, uint64_t* ticket);
/* b200_box_submit_settlement with the settlement given as a witness vector (b200_pool_submit_settlement_witness); the
 * witness counts among the job's device pointers. */
int b200_box_submit_settlement_witness(b200_box* box, const b200_box_srs* srs, const b200_box_pk* pk,
                                       const b200_bundle_witness* proof, const b200_settlement_link* links, size_t n_links,
                                       int* statuses, uint64_t* ticket);

#ifdef __cplusplus
}
#endif
#endif /* B200SETTLEMENT_H */
