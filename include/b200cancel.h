/* b200cancel.h — cancellation of libb200prover's prover pool and box jobs, by ticket or all at once.
 *
 * A relayer that is told to stop, or whose task failed after its jobs were queued (a match given up before its
 * settlement), has work on its GPUs that nobody will read.  b200_pool_destroy drains every queue first; a combined
 * verification job over attacker-chosen items bisects for tens of seconds.  These calls take jobs back instead.
 *
 * A job layer over the pool and box of b200prover.h (and the express lane of b200express.h), declared in a header of
 * its own with the same conventions (libb200prover.so), plus one error code.
 *
 * Semantics:
 *   - Queued jobs.  b200_pool_cancel removes the ticket's queued jobs from the normal queue and from the express queue;
 *     they never run.  *dropped is how many it removed (1 for a single job, up to the proof count for a bundle).
 *   - Bundles.  A cancelled bundle forks no link jobs; its queued proof or link sub-jobs are dropped.
 *   - Running jobs.  A running job is asked to stop at its next abort point: a place where the host already waits for
 *     the device (each Fiat–Shamir round trip of a proof, between the chunks of a batch, between a link proof's two
 *     segments, between a settlement's proof and its links, between a bundle's sub-jobs, between the stages and the
 *     bisection steps of a verification job).  No kernel is interrupted: the wait is at most the work up to that point.
 *     The ticket's b200_pool_wait / b200_pool_wait_info then returns B200_ERR_CANCELLED, unless the job finished before
 *     it reached an abort point: its wait then returns the status it really had.  After B200_ERR_CANCELLED the job's
 *     output buffers (proofs, link polynomials, statuses, verdicts) hold unspecified bytes: do not read them.
 *   - An aborted call leaves its worker's context as reusable as a finished one: its streams are synchronised, no
 *     capture is left open, and a partial set of captured graphs is dropped (the next proof of that key captures again).
 *   - Return codes.  Cancelling a ticket that has finished, or was cancelled already, is B200_OK with *dropped = 0.
 *     B200_ERR_INVALID for a NULL pool, box or dropped, a ticket never handed out, or one already waited for (exactly
 *     as b200_pool_expedite).
 *   - b200_pool_cancel_all does this for every ticket the pool holds.  Submits that follow it are accepted as usual:
 *     cancellation is an action, not a state of the pool.
 *   - Counters.  b200_pool_stats keeps its four counters; a cancelled job counts as completed and as failed.
 *     b200_pool_wait_all reports B200_ERR_CANCELLED for cancelled jobs not waited for individually, as for any failure.
 *     b200_pool_wait_info of a ticket whose last job was dropped from a queue reports worker (unsigned)-1: none ran it.
 *   - b200_pool_destroy and b200_box_destroy keep draining what is queued.  To stop now, call cancel_all first, then
 *     destroy: the destroy then waits at most for each worker's next abort point.
 *   - Only pool and box jobs can be cancelled: the single-context entry points (b200_plonk_prove, ...) never abort. */
#ifndef B200CANCEL_H
#define B200CANCEL_H

#include "b200prover.h"

#define B200_ERR_CANCELLED (-8) /* the job was cancelled before it finished */

#ifdef __cplusplus
extern "C" {
#endif

/* ---- on a prover pool ---------------------------------------------------------------------------------------------- */
/* Cancel the ticket's job: drop its queued jobs (*dropped of them) and ask its running ones to stop. */
int b200_pool_cancel(b200_pool* pool, uint64_t ticket, size_t* dropped);
/* b200_pool_cancel for every ticket the pool holds; *dropped is the total of jobs removed from both queues. */
int b200_pool_cancel_all(b200_pool* pool, size_t* dropped);

/* ---- on a box ------------------------------------------------------------------------------------------------------ */
/* b200_pool_cancel on the pool of the ticket's device.  B200_ERR_INVALID also for a ticket whose device index is outside
 * the box. */
int b200_box_cancel(b200_box* box, uint64_t ticket, size_t* dropped);
/* b200_pool_cancel_all on every device's pool; *dropped is the total over the devices. */
int b200_box_cancel_all(b200_box* box, size_t* dropped);

#ifdef __cplusplus
}
#endif
#endif /* B200CANCEL_H */
