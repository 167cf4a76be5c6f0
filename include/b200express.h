/* b200express.h — the express lane of libb200prover's prover pool and box: urgent jobs moved, by ticket, ahead of the
 * proof load onto reserved workers whose streams outrank it.
 *
 * A relayer has urgent work (a match's settlement proof and its link proofs, on a trade's critical path; the gossip
 * layer's order checks) and background work (validity proofs of orders being placed) on the same GPUs.  In a plain pool
 * an urgent job waits twice: on the host behind every job already queued, and on the GPU, where its long kernels share
 * the SMs with those of every other proof in flight.  b200_pool_expedite removes the first wait for a job of any kind
 * (prove, witness, batch, link, link batch, bundle, settlement, verify); express workers address the second.
 *
 * A job layer over the core ABI of b200prover.h (its pool and box), declared in a header of its own: b200prover.h stays
 * the core entry-point set, and this header adds the six express-lane entry points of the same library
 * (libb200prover.so), with the same conventions and error codes.  Pools and boxes made by b200_pool_create /
 * b200_box_create have no express workers and are expedited like any other. */
#ifndef B200EXPRESS_H
#define B200EXPRESS_H

#include "b200prover.h"

#ifdef __cplusplus
extern "C" {
#endif

/* ---- on a prover pool ---------------------------------------------------------------------------------------------- */
/* A pool of `n_workers` normal workers and `n_express` express workers on `device`, each with a context of its own.
 * Two queues: the normal FIFO every submit call appends to, and the express queue b200_pool_expedite moves jobs to.
 *   - Express workers take jobs from the express queue only, in the order the jobs were expedited.
 *   - A normal worker takes from the express queue first when it holds more jobs than there are idle express workers,
 *     else from the normal queue.  With no express workers the express queue is simply the front of the line.
 * An express context's stream of each role ranks above a normal context's of the same role, per B200_STREAM_PRIORITIES
 * (the range read with cudaDeviceGetStreamPriorityRange):
 *   unset or 1: main stream at the greatest priority (as in a normal context), the companion stream of the long kernels
 *               (accumulation, NTT passes, quotient) one level above the least instead of at the least;
 *   0:          its one stream at the greatest priority instead of 0.
 * On a device with fewer than two levels express contexts equal normal ones.  Captured graphs keep their stream's
 * priority, so an express context's graphs replay at express priority.  Priorities decide which waiting blocks the
 * scheduler starts next; blocks already running are not pre-empted.  Each express worker is one more context (its
 * buffers are allocated at its first job of each shape).
 * Express contexts are not reachable through b200_pool_ctx, and b200_pool_workers counts normal workers only; keys and
 * SRS tables made on any context of the device serve every worker.  b200_pool_stats' `queued` counts both queues;
 * b200_pool_wait_all and b200_pool_destroy drain both.  n_express = 0 is exactly b200_pool_create.
 * B200_ERR_INVALID for a NULL out, n_workers outside [1, 64] or n_express > 64; B200_ERR_NO_DEVICE without a device. */
int b200_pool_create_express(int device, unsigned n_workers, unsigned n_express, b200_pool** out);
/* Move the ticket's queued jobs, in their order, to the back of the express queue; *moved is how many it moved (1 for a
 * single job, up to the proof count for a bundle).  A bundle is also marked, so that the link proofs it forks once its
 * proofs are in go to the express queue too.  *moved is 0, with B200_OK, when the ticket's jobs have all started, have
 * all finished (waited for or not), or were expedited already.  B200_ERR_INVALID for a NULL pool or moved, a ticket
 * never handed out, or one already waited for. */
int b200_pool_expedite(b200_pool* pool, uint64_t ticket, size_t* moved);
/* b200_pool_wait (same status and message; consumes the ticket) that also returns info[0], the pool's completed count
 * (b200_pool_stats' out[1]) right after the ticket's last job finished, and info[1], the index of the worker that ran
 * that job: normal workers are 0..n_workers-1, express workers n_workers and up.  Completion order and lane placement
 * can so be checked without timing, and a caller can account latency per job.  B200_ERR_INVALID also for a NULL info. */
int b200_pool_wait_info(b200_pool* pool, uint64_t ticket, uint64_t info[2]);

/* ---- on a box ------------------------------------------------------------------------------------------------------ */
/* b200_box_create with b200_pool_create_express(device, workers_per_device, express_per_device) on every device.  Jobs
 * are routed at submit exactly as in any box. */
int b200_box_create_express(const int* devices, int n_dev, unsigned workers_per_device, unsigned express_per_device,
                            b200_box** out);
/* b200_pool_expedite on the pool of the ticket's device.  B200_ERR_INVALID also for a NULL box or a ticket whose device
 * index is outside the box. */
int b200_box_expedite(b200_box* box, uint64_t ticket, size_t* moved);
/* b200_pool_wait_info on the pool of the ticket's device: info[0] counts that pool's completions and info[1] indexes its
 * workers. */
int b200_box_wait_info(b200_box* box, uint64_t ticket, uint64_t info[2]);

#ifdef __cplusplus
}
#endif
#endif /* B200EXPRESS_H */
