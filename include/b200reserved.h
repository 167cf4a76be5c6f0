/* b200reserved.h — reserved SMs for the express lane of libb200prover's prover pool and box (b200express.h): express
 * workers on a group of SMs of their own, normal workers on the rest.
 *
 * Stream priorities (b200_pool_create_express) only decide which waiting blocks start next: an urgent proof's grids
 * still wait for the blocks of the proof load already running on every SM.  A reserved pool splits the device's SMs in
 * two with green contexts (CUDA 12.5+, in-process: no daemon, no device setting) and binds each express worker's
 * context to the first group and each normal worker's to the second, so an urgent job's blocks never queue behind the
 * load's.  The price: the reserved SMs idle while no urgent job runs.
 *
 * A job layer over the pool and box of b200prover.h and b200express.h, declared in a header of its own with the same
 * conventions and error codes (libb200prover.so).  Every express rule holds as for b200_pool_create_express: the two
 * queues, b200_pool_expedite, a normal worker taking from the express queue when it backs up, b200_pool_wait_info's
 * worker indices (normal 0..n_workers-1, express n_workers and up).  Each worker's context has a green context of its
 * own on its group (a green context is current to one thread at a time); every entry point on such a context makes it
 * current for the call and restores the caller's context after.  Memory is the device's: keys, SRS tables and buffers
 * made on any context of the device, partitioned or not, serve every worker.  Pools and boxes made by the other create
 * calls have no partition. */
#ifndef B200RESERVED_H
#define B200RESERVED_H

#include "b200prover.h"

#ifdef __cplusplus
extern "C" {
#endif

/* ---- on a prover pool ---------------------------------------------------------------------------------------------- */
/* b200_pool_create_express(device, n_workers, n_express) with the device's SMs split into an express group of at least
 * `express_sms` SMs (the split rounds up to the device's granularity) and a normal group of the rest; the n_express
 * express workers run on the first, the n_workers normal workers on the second.  Stream priorities are those of
 * b200_pool_create_express.  Nothing is created on a refusal.
 * B200_ERR_INVALID, naming the rule, for a NULL out, n_workers outside [1, 64], n_express outside [1, 64], express_sms of
 * 0, not a multiple of 8 or above 248 (a normal group of at least 8 SMs on a device of at most 256), and, on the device,
 * an express group that leaves fewer than 8 SMs for the normal one; B200_ERR_NO_DEVICE without a device; B200_ERR_CUDA
 * when the driver has no green contexts. */
int b200_pool_create_reserved(int device, unsigned n_workers, unsigned n_express, unsigned express_sms, b200_pool** out);
/* out[0] = the normal group's SM count, out[1] = the express group's, as the split rounded them; 0, 0 for a pool made
 * without a partition.  B200_ERR_INVALID for a NULL pool or out. */
int b200_pool_partition(const b200_pool* pool, unsigned out[2]);
/* A diagnostic of placement: on worker `worker`'s context (normal 0..n_workers-1, express after), a small kernel with
 * eight blocks per SM of the context runs on each of its streams, once eagerly and once as a captured and replayed
 * graph, and ORs each block's %smid into mask (bit i % 64 of mask[i / 64]; mask is zeroed first).  The context's side
 * stream exists once it has proved.  B200_ERR_INVALID for a NULL pool or mask, or a worker index out of range. */
int b200_pool_probe_sms(b200_pool* pool, unsigned worker, uint64_t mask[4]);

/* ---- on a box ------------------------------------------------------------------------------------------------------ */
/* b200_box_create with b200_pool_create_reserved(device, workers_per_device, express_per_device, express_sms) on every
 * device.  Jobs are routed at submit exactly as in any box. */
int b200_box_create_reserved(const int* devices, int n_dev, unsigned workers_per_device, unsigned express_per_device,
                             unsigned express_sms, b200_box** out);

#ifdef __cplusplus
}
#endif
#endif /* B200RESERVED_H */
