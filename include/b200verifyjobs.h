/* b200verifyjobs.h — verification jobs of libb200prover: b200_plonk_verify_each / b200_plonk_batch_verify queued on a
 * prover pool or a box, run by a worker on its own context next to the proofs, and waited for by ticket.
 *
 * The shape of the gossip layer's order check (workers/gossip-server/src/orderbook.rs:180-229: two proofs and one link
 * proof per order), which runs in the same process as the proof manager.  A pool's contexts are off limits while jobs
 * run (b200_pool_ctx), so without these jobs a caller that verifies on a proving GPU keeps a context of its own there.
 *
 * A job layer over the core ABI of b200prover.h (its verifiers, pool and box), declared in a header of its own:
 * b200prover.h stays the core entry-point set, and this header adds the two verification-job entry points of the same
 * library (libb200prover.so), with the same conventions and error codes. */
#ifndef B200VERIFYJOBS_H
#define B200VERIFYJOBS_H

#include "b200prover.h"

#ifdef __cplusplus
extern "C" {
#endif

/* ---- on a prover pool ---------------------------------------------------------------------------------------------- */
/* Queue ONE verification job on some worker of the pool (one job in b200_pool_stats):
 *   mode 0: b200_plonk_verify_each(ctx_of_that_worker, vks, n_vks, proofs, n_proofs, links, n_links, g2_h, g2_tau_h,
 *           verdicts) — every item checked with its own pairing;
 *   mode 1: b200_plonk_batch_verify(ctx_of_that_worker, ..., all_accepted, verdicts) — one combined pairing, failing
 *           items found by bisection inside the job.
 * Copied at submit: the vks array and each key's k / selector / sigma commitments, the proofs array with each item's
 * public inputs and b200_proof, the links array with each item's comm1 / comm2 and b200_link_proof, and both G2 records.
 * The caller therefore may free or reuse every input as soon as the call returns.  verdicts (n_proofs + n_links bytes,
 * proofs first) and all_accepted (mode 1; may be NULL) stay owned by the caller until the ticket has been waited for.
 * Verdicts and all_accepted are byte-for-byte the bare-context call's on the same inputs; a rejected item (malformed
 * ones included: an off-curve G1 point, a field element >= p, a public input >= r) is a verdict of 0, not an error.
 * The ticket's status is the call's status.  Zero items are accepted (the job completes with B200_OK, all_accepted 1).
 * Refused at submit, with nothing queued and b200_last_error() naming the argument or item:
 *   B200_ERR_INVALID      a NULL pool / ticket / G2 record; a NULL vks / proofs / links array with a nonzero count;
 *                         NULL verdicts when there are items; a mode other than 0 or 1; a key with log_n > 28 or a NULL
 *                         k / selector / sigma pointer; a proof with a vk index out of range, a NULL proof or NULL public
 *                         inputs for a key with inputs; a link with a NULL comm1 / comm2 / proof, alignment > 28,
 *                         size 0 or size > 2^alignment;
 *   B200_ERR_NOT_ON_CURVE a G2 record off the twist (a coordinate >= q included). */
int b200_pool_submit_verify(b200_pool* pool, int mode, const b200_verifying_key* vks, size_t n_vks,
                            const b200_batch_proof* proofs, size_t n_proofs, const b200_batch_link* links, size_t n_links,
                            const uint64_t g2_h[16], const uint64_t g2_tau_h[16], int* all_accepted, uint8_t* verdicts,
                            uint64_t* ticket);

/* ---- on a box ------------------------------------------------------------------------------------------------------ */
/* b200_pool_submit_verify on the least-loaded device of the box.  Every input is copied to the host at submit, so no
 * job is pinned to a device.  Tickets are waited for with b200_box_wait; b200_box_ticket_device names the device.
 * Refusals as b200_pool_submit_verify (a NULL box included). */
int b200_box_submit_verify(b200_box* box, int mode, const b200_verifying_key* vks, size_t n_vks,
                           const b200_batch_proof* proofs, size_t n_proofs, const b200_batch_link* links, size_t n_links,
                           const uint64_t g2_h[16], const uint64_t g2_tau_h[16], int* all_accepted, uint8_t* verdicts,
                           uint64_t* ticket);

#ifdef __cplusplus
}
#endif
#endif /* B200VERIFYJOBS_H */
